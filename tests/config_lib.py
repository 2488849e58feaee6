"""The numeric range of serfsim_config_t, shared by tests/test_config_envelope.py and tests/test_gpu_z_config_envelope.py — test
infrastructure only.

- config_fuzz: envelope_lib.envelope_fuzz with every config field drawn over the whole range serfsim_create accepts, weighted
  towards the edges (k up to 7, budgets up to 255, clocks a few hundred below the Lamport limit, n at powers of ten ± 1).
- expected_retransmit_limit / expected_suspicion_table: a restatement of the two derived constants in Python, independent of both
  C++ copies (serf_b200/csrc/serfsim.cu and oracle/serf_oracle.cpp).  exact_suspicion_entries gives the entries that exact
  rational arithmetic fixes without any floating point.
- accepted: the validation rule of serfsim_create as a predicate (DESIGN.md §2 rule 10).
- LTIME_LIMIT, INC_LIMIT, MAX_K: read from serf_b200/csrc/record.cuh.
"""
import math
import os
import re
from fractions import Fraction

import numpy as np

import envelope_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _record_constant(name):
    src = open(os.path.join(ROOT, "serf_b200", "csrc", "record.cuh")).read()
    m = re.search(r"constexpr u32 " + name + r" = ([^;]+);", src)
    assert m, name
    expr = re.sub(r"(0x[0-9A-Fa-f]+|\d+)u\b", r"\1", m.group(1))
    assert re.fullmatch(r"[0-9A-Fa-fx()<\-+ ]+", expr), expr
    return int(eval(expr))                                      # noqa: S307 — digits, shifts and +/- only (checked above)


LTIME_LIMIT = _record_constant("LTIME_LIMIT")
INC_LIMIT = _record_constant("INC_LIMIT")
MAX_K = _record_constant("MAX_K")
INIT_LTIME_BOUND = LTIME_LIMIT - 16           # init_clock / init_status_ltime must be below this
TIMEOUT_LIMIT = 1 << 30                       # largest suspicion timeout in ticks
INT64_MAX = (1 << 63) - 1
U32_MAX = (1 << 32) - 1
GOSSIP_MS = (1, 3, 7, 199, 200, 201, 999, 1000, 4999)
DECADE_EDGES = (9, 10, 11, 99, 100, 101, 999, 1000, 1001)


# ---- the derived constants, restated -------------------------------------------------------------------------
def digits(n):
    """ceil(log10(n + 1)) in exact integers: the smallest d with 10^d >= n + 1."""
    d, p = 0, 1
    while p < n + 1:
        p *= 10
        d += 1
    return d


def expected_retransmit_limit(mult, n):
    """memberlist's retransmit limit, retransmit_mult · ceil(log10(n + 1)), as an unbounded integer."""
    return mult * digits(n)


def _ms(susp_mult, max_mult, probe_ticks, tick_ms, n):
    """(min_ms, max_ms, the product before the division) in exact integers; node_scale goes through the double log10 as upstream."""
    node_scale = max(1.0, math.log10(max(1.0, float(n))))
    prod = susp_mult * int(node_scale * 1000.0) * (probe_ticks * tick_ms)
    min_ms = prod // 1000
    return min_ms, max_mult * min_ms, prod


def suspicion_k(susp_mult, n):
    k = susp_mult - 2
    if n - 2 < k:
        k = 0
    return max(k, 0)


def expected_suspicion_table(susp_mult, max_mult, probe_ticks, tick_ms, n):
    """Lifeguard's suspicion timeouts in ticks: min = suspicion_mult · max(1, log10 n) · probe interval (ms, as
    mult · int(node_scale · 1000) · interval / 1000), max = suspicion_max_timeout_mult · min, k = suspicion_mult − 2 (0 when
    n − 2 < k); entry c = floor(max − log(c+1)/log(k+1) · (max − min)) ms, at least min, then ceil(ms / tick_ms), at least 1.
    The formula is defined in double arithmetic: Python floats are the same IEEE doubles."""
    min_ms, max_ms, _ = _ms(susp_mult, max_mult, probe_ticks, tick_ms, n)
    k = suspicion_k(susp_mult, n)
    out = []
    for c in range(k + 1):
        if k < 1:
            ms = min_ms
        else:
            frac = math.log(c + 1.0) / math.log(k + 1.0)
            ms = max(math.floor(float(max_ms) - frac * float(max_ms - min_ms)), min_ms)
        out.append(max(1, -(-ms // tick_ms)))
    return out


def exact_scale_milli(n):
    """int(max(1, log10 n) · 1000) where exact arithmetic fixes it (n ≤ 10 or n a power of ten), else None."""
    if n <= 10:
        return 1000
    d = digits(n) - 1
    return 1000 * d if 10 ** d == n else None


def exact_suspicion_entries(susp_mult, max_mult, probe_ticks, tick_ms, n):
    """{c: ticks} for the entries exact rational arithmetic fixes without floating point: all of them when k < 1 or
    max = min (suspicion_max_timeout_mult 0 or 1), else c = 0 (log 1 = 0: the max) and c = k (the fraction is 1: the min).
    Needs a node count whose log10 is exact and ms values below 2^53 (where doubles hold every integer)."""
    milli = exact_scale_milli(n)
    if milli is None:
        return {}
    min_ms = Fraction(susp_mult * milli * probe_ticks * tick_ms, 1000).__floor__()
    max_ms = max_mult * min_ms
    if max(min_ms, max_ms) >= 1 << 53:
        return {}
    ceil_ticks = lambda ms: max(1, -(-ms // tick_ms))
    k = suspicion_k(susp_mult, n)
    if k < 1 or max_mult <= 1:
        return {c: ceil_ticks(min_ms) for c in range(k + 1)}
    return {0: ceil_ticks(max(max_ms, min_ms)), k: ceil_ticks(min_ms)}


# ---- the validation rule of serfsim_create ----------------------------------------------------------------------
def rejection(cfg, n=None):
    """None when serfsim_create accepts the numeric fields of `cfg` (a dict or a sim.Config; n defaults to n_nodes), else the
    name of the first field the product's message must name.  Topology-shaped fields (slots, fan-out, world) are not covered."""
    g = (lambda f: cfg[f]) if isinstance(cfg, dict) else (lambda f: getattr(cfg, f))
    n = g("n_nodes") if n is None else n
    if g("gossip_interval_ms") == 0:
        return "gossip_interval_ms"
    if g("suspicion_mult") > MAX_K + 2:
        return "suspicion_mult"
    if g("init_clock") >= INIT_LTIME_BOUND:
        return "init_clock"
    if g("init_status_ltime") >= INIT_LTIME_BOUND:
        return "init_status_ltime"
    if not 1 <= expected_retransmit_limit(g("retransmit_mult"), n) <= 255:
        return "retransmit_mult"
    probe = g("probe_interval_ticks") or 1
    tick_ms, susp, mx = g("gossip_interval_ms"), g("suspicion_mult"), g("suspicion_max_timeout_mult")
    min_ms, max_ms, prod = _ms(susp, mx, probe, tick_ms, n)
    if probe * tick_ms > INT64_MAX or prod > INT64_MAX:
        return "gossip_interval_ms"
    if max_ms > INT64_MAX:
        return "suspicion_max_timeout_mult"
    top = max(min_ms, max_ms) if suspicion_k(susp, n) >= 1 else min_ms        # k < 1: the table is the minimum alone
    if -(-top // tick_ms) > TIMEOUT_LIMIT or max(expected_suspicion_table(susp, mx, probe, tick_ms, n)) > TIMEOUT_LIMIT:
        return "suspicion_max_timeout_mult"
    return None


def accepted(cfg, n=None):
    return rejection(cfg, n) is None


# ---- the fuzzer -------------------------------------------------------------------------------------------------
def _edge_int(rng, lo, hi, edges=()):
    """An integer in [lo, hi]: half of the time one of the ends or `edges`, otherwise uniform."""
    if rng.random() < 0.5:
        pool = [x for x in (lo, hi, *edges) if lo <= x <= hi]
        return int(pool[int(rng.integers(0, len(pool)))])
    return int(rng.integers(lo, hi + 1))


def config_fuzz(seed, n=None):
    """envelope_lib.envelope_fuzz (every operation kind, fan-out 1–8, slots 1–16, regular / small-world / irregular graphs) with
    every config field drawn over what serfsim_create accepts.  The node count is sometimes a power of ten ± 1 (where the
    retransmit limit and the node scale step) and sometimes small enough that n − 2 < k.  Lamport times start up to a few hundred
    below the validation bound: far enough from LTIME_LIMIT that the run's few hundred increments stay below it (the test checks
    that on the oracle).  The same seed gives the same scenario everywhere."""
    rng = np.random.Generator(np.random.Philox(seed + 31_000_017))
    susp = _edge_int(rng, 0, MAX_K + 2, (2, 3))
    if n is None:
        r = rng.random()
        if r < 0.3:
            n = int(DECADE_EDGES[int(rng.integers(0, len(DECADE_EDGES) - 3))])       # 999–1001 only when asked for: slow on the host build
        elif r < 0.45:
            n = int(rng.integers(3, max(4, min(susp, 9))))                            # n - 2 < k whenever susp > 3
    sc = envelope_lib.envelope_fuzz(seed, n=n)
    n = sc.n
    d = digits(n)
    cfg = sc.cfg
    cfg.update(suspicion_mult=susp,
               suspicion_max_timeout_mult=_edge_int(rng, 0, 10, (1,)),
               probe_interval_ticks=_edge_int(rng, 0, 12, (1,)),
               gossip_interval_ms=int(GOSSIP_MS[int(rng.integers(0, len(GOSSIP_MS)))]),
               retransmit_mult=_edge_int(rng, 1, 255 // d),
               reap_interval_ticks=_edge_int(rng, 0, 25, (1,)),
               tombstone_timeout_ticks=_edge_int(rng, 0, 80, (1,)),
               reconnect_timeout_ticks=_edge_int(rng, 0, 80, (1,)),
               recent_intent_timeout_ticks=_edge_int(rng, 0, 80, (1,)),
               push_pull_interval_ticks=int(rng.choice([0, 0, 1, 2, 5, 11, 30])))
    for f, small in (("init_clock", (1, 5)), ("init_status_ltime", (0, 3))):
        cfg[f] = INIT_LTIME_BOUND - int(rng.integers(300, 700)) if rng.random() < 0.3 else int(rng.integers(*small))
    assert accepted(dict(cfg, n_nodes=n)), (seed, cfg)
    sc.name = f"config_fuzz_{seed}_n{n}"
    return sc


def max_ltime(o, slots):
    """The largest Lamport time a simulator holds: clocks, status times (buffered intent times included) and queued intent times."""
    m = int(o.lamport_time().max())
    for s in range(slots):
        r = o.records(s)
        m = max(m, int(r["status_ltime"].max()), int(r["qjoin_lt"].max()), int(r["qleave_lt"].max()))
    return m
