"""The configuration range the other parity tests never draw, on the CPU: the derived constants (retransmit limit, suspicion
timeouts) against an independent restatement, the product's own timeout table pinned end to end through the host build of the
kernels (tests/emu), config_fuzz against the oracle, the validation rule of serfsim_create, and the SERFSIM_E_OVERFLOW contract
at the Lamport limit.

Not covered: incarnations near INC_LIMIT.  No config sets them, and reaching 2^26 refutations in a test run is not practical.
The user-event path's event clock cannot be driven to the limit either: it starts at 1 and only the (at most 8) tracked events
raise it, so the overflow runs below cover the member clocks, status times and queued intent times.
"""
import ctypes as C
import threading

import numpy as np
import pytest

import config_lib as CL
import parity_lib as P
from emu_lib import emu_sim
from oracle_lib import lib as olib, oracle_sim
from serf_b200 import MlState, scenarios
from serf_b200.scenarios import Op, Scenario
from serf_b200.sim import SerfsimError, full_mesh_graph, random_regular_graph

E_INVAL, E_OVERFLOW = -1, -5


def oracle_table(susp, mx, probe, tick_ms, n):
    out = (C.c_uint32 * 8)()
    k = olib().oracle_suspicion_table(susp, mx, probe, tick_ms, n, out, 8)
    return list(out[:k])


def _largest_probe(susp, mx, tick_ms, n):
    """The largest probe_interval_ticks (≤ 2^32 − 1) whose table serfsim_create accepts at this tick length."""
    cfg = dict(n_nodes=n, suspicion_mult=susp, suspicion_max_timeout_mult=mx, gossip_interval_ms=tick_ms, retransmit_mult=1,
               init_clock=2, init_status_ltime=1)
    lo, hi = 1, CL.U32_MAX
    if CL.accepted(dict(cfg, probe_interval_ticks=hi)):
        return hi
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if CL.accepted(dict(cfg, probe_interval_ticks=mid)) else (lo, mid)
    return lo


NODE_EDGES = sorted({2, 3, 8, 9} | {x for e in range(1, 8) for x in (10 ** e - 1, 10 ** e, 10 ** e + 1)} | {1 << 26})


# ---- the derived constants ---------------------------------------------------------------------------------------
def test_retransmit_limit_restated_at_every_decade_edge():
    for n in NODE_EDGES:
        assert CL.digits(n) == len(str(n))                      # ceil(log10(n + 1)) is the number of decimal digits
        for mult in (1, 2, 3, 4, 31, 63, 85, 127, 255):
            want = CL.expected_retransmit_limit(mult, n)
            assert olib().oracle_retransmit_limit(mult, n) == want, (mult, n)
    assert CL.digits(9) == 1 and CL.digits(10) == 2 and CL.digits(99) == 2 and CL.digits(100) == 3 and CL.digits(1 << 26) == 8


def test_suspicion_table_restated_on_the_grid():
    """Every suspicion_mult 0–9 and suspicion_max_timeout_mult 0–10, probe × tick products from 1 to the largest accepted, n at
    every decade edge: the Python table equals the oracle's, and every entry exact rational arithmetic fixes is what it says."""
    pairs = [(1, 1), (1, 3), (2, 7), (5, 200), (3, 201), (12, 4999), (1, 199), (7, 999), (12, 1)]
    compared = exact = 0
    for n in NODE_EDGES:
        for susp in range(0, CL.MAX_K + 3):
            for mx in range(0, 11):
                grid = list(pairs)
                for tick_ms in (1, 200, 4999, CL.U32_MAX):
                    p = _largest_probe(susp, mx, tick_ms, n)
                    grid.append((p, tick_ms))
                for probe, tick_ms in grid:
                    cfg = dict(n_nodes=n, suspicion_mult=susp, suspicion_max_timeout_mult=mx, probe_interval_ticks=probe,
                               gossip_interval_ms=tick_ms, retransmit_mult=1, init_clock=2, init_status_ltime=1)
                    if not CL.accepted(cfg):
                        continue
                    want = CL.expected_suspicion_table(susp, mx, probe, tick_ms, n)
                    assert len(want) == CL.suspicion_k(susp, n) + 1
                    assert oracle_table(susp, mx, probe, tick_ms, n) == want, (susp, mx, probe, tick_ms, n)
                    assert max(want) <= CL.TIMEOUT_LIMIT
                    if max(CL._ms(susp, mx, probe, tick_ms, n)[:2]) < 1 << 53:       # above 2^53 ms the double step may round up by one
                        assert all(a >= b for a, b in zip(want, want[1:])), (susp, mx, probe, tick_ms, n, want)
                    compared += 1
                    for c, t in CL.exact_suspicion_entries(susp, mx, probe, tick_ms, n).items():
                        assert want[c] == t, (susp, mx, probe, tick_ms, n, c)
                        exact += 1
    assert compared > 20_000 and exact > 20_000, (compared, exact)
    # the LAN profile at 100 K nodes, by hand: min = 4 · 5 · 1 s = 20 s = 100 ticks, max = 6 · min = 600 ticks, and the middle
    # entry 120 s − log 2 / log 3 · 100 s = 56.907 s = 284.5 ticks, rounded up
    assert CL.expected_suspicion_table(4, 6, 5, 200, 100_000) == [600, 285, 100]


def test_n_below_k_drops_the_confirmations():
    for susp in range(3, CL.MAX_K + 3):
        k = susp - 2
        for n in (3, k + 1, k + 2):
            t = CL.expected_suspicion_table(susp, 6, 1, 200, n)
            assert len(t) == (1 if n - 2 < k else k + 1)
            assert oracle_table(susp, 6, 1, 200, n) == t


# ---- the product's own table, end to end ----------------------------------------------------------------------------
def test_product_timeout_table_pinned_by_the_confirmation_deadlines():
    """k = 7 (suspicion_mult 9): a crash at tick 0 in a full mesh where every node probes every tick.  A view that became Suspect
    at tick t0 and holds c confirmations (popcount(mask) = c + 1 confirmer buckets) has deadline t0 + table[c], so
    deadline − t0 pins every entry of the product's table (h->rules.timeout) against the Python restatement, without the oracle.
    A 1 ms tick makes ticks equal milliseconds, so each interior entry is the floored double of the formula itself."""
    n, susp, mx, probe, tick_ms = 64, 9, 10, 1, 1
    table = CL.expected_suspicion_table(susp, mx, probe, tick_ms, n)
    assert len(table) == 8 and len(set(table)) == 8
    sc = Scenario("lifeguard_k7", n, 1, full_mesh_graph(n), [3], [(0, Op.FAIL, 3, 0)],
                  dict(fanout=3, seed=5, suspicion_mult=susp, suspicion_max_timeout_mult=mx, probe_interval_ticks=probe,
                       gossip_interval_ms=tick_ms))
    for trace in (1, 0):
        g = sc.build(emu_sim, trace=trace)
        t0 = np.full(n, -1, dtype=np.int64)
        seen = set()
        checked = 0
        for _ in range(table[0] + 2):
            g.step(1)
            t = g.stats()["tick"] - 1                             # the tick just executed
            r = g.records(0)
            sus = (r["ml"] & 3) == MlState.SUSPECT
            t0[sus & (t0 < 0)] = t
            for v in np.nonzero(sus & (r["deadline"] != 0))[0]:
                c = bin(int(r["conf_mask"][v])).count("1") - 1
                assert int(r["deadline"][v]) - int(t0[v]) == table[c], (trace, v, t, c)
                seen.add(c)
                checked += 1
        assert seen == set(range(8)), seen                        # every entry was reached, the full set of 8 confirmers too
        assert checked > 500
        assert ((g.records(0)["ml"] & 3) == MlState.DEAD).sum() > 0


# ---- config_fuzz against the oracle ---------------------------------------------------------------------------------
def _parity_or_overflow(sc):
    o = sc.build(oracle_sim, trace=1)
    o.run_until_converged(sc.max_ticks)
    assert CL.max_ltime(o, sc.slots) < CL.LTIME_LIMIT, sc.name        # the draw keeps every run inside the device range
    P.run_against_oracle(emu_sim, sc)
    return o


FUZZ_SEEDS = range(24)


@pytest.mark.parametrize("seed", FUZZ_SEEDS)
def test_config_fuzz(seed):
    _parity_or_overflow(CL.config_fuzz(seed))


def test_config_fuzz_reaches_the_edges():
    """What test_config_fuzz claims to cover is drawn by its seeds."""
    scs = [CL.config_fuzz(s) for s in FUZZ_SEEDS]
    assert {sc.n for sc in scs} & set(CL.DECADE_EDGES)
    assert any(sc.n - 2 < sc.cfg["suspicion_mult"] - 2 for sc in scs)
    assert any(sc.cfg["suspicion_mult"] == 9 for sc in scs) and any(sc.cfg["suspicion_mult"] == 0 for sc in scs)
    assert any(CL.expected_retransmit_limit(sc.cfg["retransmit_mult"], sc.n) >= 248 for sc in scs)
    assert any(sc.cfg["init_clock"] > CL.LTIME_LIMIT - 1000 for sc in scs) and any(sc.cfg["init_status_ltime"] > CL.LTIME_LIMIT - 1000 for sc in scs)
    assert {sc.cfg["gossip_interval_ms"] for sc in scs} >= {1, 4999}
    assert any(sc.cfg["push_pull_interval_ticks"] == 1 for sc in scs) and any(sc.cfg["tombstone_timeout_ticks"] == 0 for sc in scs)


@pytest.mark.parametrize("n", CL.DECADE_EDGES)
def test_config_fuzz_at_a_power_of_ten(n):
    """n = 10^k − 1, 10^k, 10^k + 1: where the retransmit limit gains a digit and the node scale log10 n is exact."""
    _parity_or_overflow(CL.config_fuzz(500 + n, n=n))


@pytest.mark.parametrize("seed,n", [(1, 101), (2, 1001), (3, 1001)])
def test_config_fuzz_sharded_across_a_power_of_ten(seed, n):
    """Two ranks of N = 10^k + 1 nodes: each shard holds fewer than 10^k, so a retransmit limit derived from the shard size
    instead of N would be one digit short."""
    sc = CL.config_fuzz(seed, n=n)
    sc.max_ticks = 200
    assert CL.digits((n + 1) // 2) == CL.digits(n) - 1
    P.run_against_oracle(emu_sim, sc, world=2)


# ---- validation ---------------------------------------------------------------------------------------------------
def _create(n=1000, **kw):
    g = emu_sim(n, 1, **kw)
    g.close()


def _rejected(field, n=1000, **kw):
    assert CL.rejection(dict(CL_DEFAULTS, n_nodes=n, **kw)) == field, (field, kw)
    with pytest.raises(SerfsimError) as ei:
        _create(n, **kw)
    assert ei.value.code == E_INVAL and field in str(ei.value), str(ei.value)


def _accepted(n=1000, **kw):
    assert CL.accepted(dict(CL_DEFAULTS, n_nodes=n, **kw)), kw
    _create(n, **kw)


CL_DEFAULTS = dict(retransmit_mult=4, suspicion_mult=4, suspicion_max_timeout_mult=6, probe_interval_ticks=5, gossip_interval_ms=200,
                   init_status_ltime=1, init_clock=2)


def test_bootstrap_lamport_times_below_the_bound():
    b = CL.INIT_LTIME_BOUND
    assert b == 0x7FFFFFE0
    for f in ("init_clock", "init_status_ltime"):
        _accepted(**{f: b - 1})
        for v in (b, CL.LTIME_LIMIT - 1, CL.LTIME_LIMIT, 0xFFFFFFFF):
            _rejected(f, **{f: v})


def test_retransmit_limit_in_64_bits():
    _accepted(n=1000, retransmit_mult=63)                     # 252
    _rejected("retransmit_mult", n=1000, retransmit_mult=64)
    _accepted(n=999, retransmit_mult=85)                      # 255
    _rejected("retransmit_mult", n=999, retransmit_mult=86)
    _rejected("retransmit_mult", n=1000, retransmit_mult=0)
    _rejected("retransmit_mult", n=1000, retransmit_mult=0x40000001)     # 4 in u32
    _rejected("retransmit_mult", n=10, retransmit_mult=0x80000000)       # 0 in u32
    _accepted(n=9, retransmit_mult=255)


def test_suspicion_timeouts_representable():
    # the confirmed case: a 12 · 2^30-tick first timeout used to come out as [0, 460466627, 12]
    _rejected("suspicion_max_timeout_mult", n=1000, suspicion_mult=4, suspicion_max_timeout_mult=0x40000000, probe_interval_ticks=1)
    # ms arithmetic beyond int64: the product, then the max multiplier
    _rejected("gossip_interval_ms", n=1000, suspicion_mult=9, probe_interval_ticks=0xFFFFFFFF, gossip_interval_ms=0xFFFFFFFF)
    _rejected("suspicion_max_timeout_mult", n=5, suspicion_mult=1, suspicion_max_timeout_mult=0xFFFFFFFF, probe_interval_ticks=0xFFFFFFFF,
              gossip_interval_ms=4999)
    # the largest accepted timeouts and their neighbours, for several shapes of the table
    for susp, mx, tick_ms, n in ((4, 6, 200, 1000), (9, 10, 1, 64), (2, 0, 4999, 10), (1, 3, 7, 100), (9, 1, 0xFFFFFFFF, 1001)):
        p = _largest_probe(susp, mx, tick_ms, n)
        kw = dict(suspicion_mult=susp, suspicion_max_timeout_mult=mx, gossip_interval_ms=tick_ms)
        _accepted(n=n, probe_interval_ticks=p, **kw)
        if tick_ms != CL.U32_MAX:                              # (at the longest tick the ms arithmetic is the bound, not the ticks)
            assert max(CL.expected_suspicion_table(susp, mx, p, tick_ms, n)) > CL.TIMEOUT_LIMIT // 2
        if p < CL.U32_MAX:
            _rejected(CL.rejection(dict(CL_DEFAULTS, n_nodes=n, probe_interval_ticks=p + 1, **kw)), n=n, probe_interval_ticks=p + 1, **kw)


def test_create_accepts_exactly_what_the_rule_accepts():
    rng = np.random.Generator(np.random.Philox(77))
    edge = lambda hi: int(rng.choice([0, 1, 2, hi, hi - 1, int(rng.integers(0, hi + 1)), int(rng.integers(0, 64))]))
    n_rej = n_acc = 0
    for _ in range(400):
        n = int(rng.choice([2, 9, 10, 11, 999, 1000, 1001, int(rng.integers(2, 5000))]))
        kw = dict(retransmit_mult=edge(0xFFFFFFFF) if rng.random() < 0.3 else int(rng.integers(0, 90)),
                  suspicion_mult=int(rng.integers(0, 12)), suspicion_max_timeout_mult=edge(0xFFFFFFFF) if rng.random() < 0.3 else int(rng.integers(0, 11)),
                  probe_interval_ticks=edge(0xFFFFFFFF) if rng.random() < 0.3 else int(rng.integers(0, 13)),
                  gossip_interval_ms=edge(0xFFFFFFFF) if rng.random() < 0.3 else int(rng.choice(CL.GOSSIP_MS)),
                  init_clock=int(rng.choice([2, CL.INIT_LTIME_BOUND - 1, CL.INIT_LTIME_BOUND, 0xFFFFFFFF])) if rng.random() < 0.2 else 2,
                  init_status_ltime=int(rng.choice([1, CL.INIT_LTIME_BOUND - 1, CL.INIT_LTIME_BOUND])) if rng.random() < 0.2 else 1)
        why = CL.rejection(dict(kw, n_nodes=n))
        if why is None:
            _create(n, **kw)
            n_acc += 1
        else:
            with pytest.raises(SerfsimError) as ei:
                _create(n, **kw)
            assert ei.value.code == E_INVAL and why in str(ei.value), (kw, n, str(ei.value))
            n_rej += 1
    assert n_acc > 100 and n_rej > 100, (n_acc, n_rej)


# ---- the overflow contract ------------------------------------------------------------------------------------------
def overflow_scenario(n=120, slots=1, init_clock=None, init_status_ltime=None, seed=3, horizon=120, push_pull=3):
    """Operations every tick that keep raising the Lamport clocks: the subjects leave and join again, other nodes force-leave
    live subjects (each one refutes with a fresh join intent), and push-pull rounds every `push_pull` ticks."""
    rng = np.random.Generator(np.random.Philox(seed))
    subjects = (np.arange(slots) * (n // slots) + 5).astype(np.uint32)
    ops = []
    for t in range(horizon):
        s = t % slots
        kind = (Op.LEAVE, Op.JOIN, Op.FORCE_LEAVE)[t % 3]
        node = int(subjects[s]) if kind != Op.FORCE_LEAVE else int((int(subjects[s]) + 1 + rng.integers(0, n - 2)) % n)
        if kind == Op.FORCE_LEAVE and node in set(int(x) for x in subjects):
            node = (node + 1) % n if (node + 1) % n not in set(int(x) for x in subjects) else (node + 2) % n
        ops.append((t, int(kind), node, s))
    cfg = dict(fanout=3, seed=seed, push_pull_interval_ticks=push_pull, suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)
    cfg["init_clock"] = CL.INIT_LTIME_BOUND - 1 if init_clock is None else init_clock
    if init_status_ltime is not None:
        cfg["init_status_ltime"] = init_status_ltime
    return Scenario(f"overflow_{n}_r{slots}", n, slots, random_regular_graph(n, 8, seed + 1), subjects, ops, cfg, max_ticks=horizon)


def overflow_step(sc, cap=None):
    """The step (1-based) after which the oracle first holds a Lamport time ≥ LTIME_LIMIT.  The oracle keeps u32 values that are
    exact until the limit; the product must fail that step with SERFSIM_E_OVERFLOW."""
    o = sc.build(oracle_sim, trace=1)
    for k in range(1, (cap or sc.max_ticks) + 1):
        o.step(1)
        if CL.max_ltime(o, sc.slots) >= CL.LTIME_LIMIT:
            return k
    raise AssertionError(f"{sc.name}: no Lamport time reached the limit in {cap or sc.max_ticks} steps")


def assert_overflow_at(sc, trace, factory=emu_sim):
    """Lockstep with the oracle: every step before the predicted one succeeds and matches it; that one fails with E_OVERFLOW."""
    k = overflow_step(sc)
    assert k > 3, k                                            # the run starts inside the range and gets there by its own operations
    o = sc.build(oracle_sim, trace=1)
    g = sc.build(factory, trace=trace)
    for i in range(k - 1):
        o.step(1)
        g.step(1)
        P.assert_same(P.outputs(g, sc, None), P.outputs(o, sc, None), with_hash=bool(trace), what=f"step {i + 1}")
    assert CL.max_ltime(g, sc.slots) < CL.LTIME_LIMIT
    with pytest.raises(SerfsimError) as ei:
        g.step(1)
    assert ei.value.code == E_OVERFLOW, str(ei.value)
    return k


@pytest.mark.parametrize("trace", [1, 0])
@pytest.mark.parametrize("slots", [1, 3])
def test_overflow_at_the_predicted_step_from_the_clock(trace, slots):
    assert_overflow_at(overflow_scenario(slots=slots), trace)


@pytest.mark.parametrize("trace", [1, 0])
@pytest.mark.parametrize("slots", [1, 3])
def test_overflow_at_the_predicted_step_from_the_status_times(trace, slots):
    """Bootstrap status times just below the bound and small clocks: the clocks get there by witnessing status times in push-pull
    rounds and intents."""
    assert_overflow_at(overflow_scenario(slots=slots, init_clock=2, init_status_ltime=CL.INIT_LTIME_BOUND - 1, seed=8), trace)


@pytest.mark.parametrize("trace", [1, 0])
@pytest.mark.parametrize("slots", [1, 3])
def test_overflow_from_gossip_alone(trace, slots):
    """No push-pull rounds: the limit is crossed in the tick kernel's own node path."""
    assert_overflow_at(overflow_scenario(slots=slots, push_pull=0, seed=21), trace)


def test_overflow_after_a_prune_and_a_crash():
    """The same contract with pruning force-leaves and crashed nodes in the mix (a crashed node's clock is frozen)."""
    sc = overflow_scenario(n=150, slots=2, seed=11)
    sc.ops = [(t, int(Op.FORCE_LEAVE_PRUNE) if op == Op.FORCE_LEAVE and t % 2 else op, node, s) for (t, op, node, s) in sc.ops]
    sc.ops += [(1, int(Op.FAIL), 77, 0), (9, int(Op.REJOIN), 77, 0)]
    for trace in (1, 0):
        assert_overflow_at(sc, trace)


def test_overflow_sharded_world_2():
    sc = overflow_scenario(n=301, slots=2, seed=4)
    k = overflow_step(sc)
    o = sc.build(oracle_sim, trace=1)
    o.step(k - 1)
    for trace in (1, 0):
        comm, world = P.ThreadComm(2), 2
        first_err, res, errs = [None, None], [None, None], []

        def worker(rank):
            try:
                g = sc.build(emu_sim, rank=rank, world_size=world, trace=trace)
                g.connect(*comm.hooks(rank))
                for i in range(1, k + 1):
                    try:
                        g.step(1)
                    except SerfsimError as e:             # keep stepping: the other rank's collectives need this one
                        if first_err[rank] is None:
                            first_err[rank] = (i, e.code)
                    if i == k - 1:
                        res[rank] = P.outputs(g, sc, None)
                comm.bar.wait()
            except BaseException as e:                    # noqa: BLE001 — surface it in the main thread
                errs.append(e)
                comm.bar.abort()
        th = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
        for t in th:
            t.start()
        for t in th:
            t.join(600)
        if errs:
            raise errs[0]
        P.assert_same(P.merge_ranks(res), P.outputs(o, sc, None), with_hash=bool(trace))
        got = [e for e in first_err if e is not None]
        assert got and all(e == (k, E_OVERFLOW) for e in got), (first_err, k)
