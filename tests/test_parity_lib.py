"""The shared parity check itself (parity_lib): two oracle runs of one scenario pass it, a copy with any single output changed or
removed fails it, and merge_ranks puts a run split into shards back together."""
import functools

import numpy as np
import pytest

import parity_lib as P
from oracle_lib import oracle_sim
from serf_b200 import scenarios

KEYS = ("run", "stats", "trace", "state_hash", "lamport_time", "lamport_time_u32", "records", "member_status", "status_ltime",
        "status_ltime_u32", "incarnation", "ml_state", "user_event_records", "user_event_stats", "event_time", "user_event_ltime",
        "user_event_seen", "byzantine_stats", "anomaly_flags")


def scenario():
    sc = scenarios.fuzz_features(1, n=300, slots=2)               # user events and injectors
    sc.max_ticks = 300
    return sc


def oracle_run():
    sc = scenario()
    o = sc.build(oracle_sim, trace=1)
    return P.outputs(o, sc, o.run_until_converged(sc.max_ticks))


@functools.lru_cache(None)
def ref():
    return oracle_run()


def changed(v):
    """Copies of v, each with one element changed (every entry of a dict, the last slot / event of a list)."""
    if isinstance(v, dict):
        return [dict(v, **{k: x + 1}) for k, x in v.items()]
    if isinstance(v, list):
        return [v[:-1] + [c] for c in changed(v[-1])]
    if isinstance(v, tuple):
        return [(v[0] + 1,) + v[1:]]
    if isinstance(v, np.ndarray):
        v = v.copy()
        field = v[v.dtype.names[0]] if v.dtype.names else v
        field[len(v) // 2] += 1
        return [v]
    return [v + 1]


def test_outputs_have_every_key():
    assert set(ref()) == set(KEYS)
    assert len(ref()["user_event_seen"]) == len(scenario().user_events) and len(ref()["records"]) == scenario().slots


def test_two_oracle_runs_agree():
    P.assert_same(oracle_run(), ref(), with_hash=True)


@pytest.mark.parametrize("key", KEYS)
def test_one_changed_element_fails(key):
    for v in changed(ref()[key]):
        with pytest.raises(AssertionError):
            P.assert_same(dict(ref(), **{key: v}), ref(), with_hash=True)


@pytest.mark.parametrize("key", KEYS)
def test_a_missing_output_fails(key):
    got = dict(ref())
    del got[key]
    with pytest.raises(AssertionError):
        P.assert_same(got, ref(), with_hash=True)
    with pytest.raises(AssertionError):
        P.assert_same(ref(), got, with_hash=True)


def test_every_trace_column_is_compared():
    trace = ref()["trace"]
    for col in trace.dtype.names:
        t = trace.copy()
        t[col][len(t) // 2] += 1
        with pytest.raises(AssertionError):
            P.assert_same(dict(ref(), trace=t), ref(), with_hash=True)
        if col == "hash":
            P.assert_same(dict(ref(), trace=t), ref(), with_hash=False)     # production mode computes no per-tick hash


def split(out, cut):
    """out as the two ranks of a sharded run whose first shard holds `cut` nodes would report it."""
    ranks = [dict(out), dict(out)]
    for k in P.PER_NODE:
        v = out[k]
        if isinstance(v, list):
            ranks[0][k], ranks[1][k] = [x[:cut] for x in v], [x[cut:] for x in v]
        else:
            ranks[0][k], ranks[1][k] = v[:cut], v[cut:]
    ranks[0]["user_event_stats"] = dict(out["user_event_stats"], event_time=0)
    return ranks


def test_merge_ranks():
    ranks = split(ref(), 137)
    ranks[1]["stats"] = dict(ranks[1]["stats"], member_time=0)               # the agreement summary is per shard
    P.assert_same(P.merge_ranks(ranks), ref(), with_hash=True)
    for key in ("run", "trace", "state_hash", "byzantine_stats", "user_event_ltime", "stats", "user_event_stats"):
        for v in changed(ref()[key]):
            if key == "stats" and any(v[k] != ref()[key][k] for k in P.SHARD_STATS):
                continue
            bad = split(ref(), 137)
            bad[1][key] = v                                                 # one rank disagrees
            with pytest.raises(AssertionError):
                P.assert_same(P.merge_ranks(bad), ref(), with_hash=True)
