"""Handle lifetime on the host build (tests/emu): a closed handle has released every device and mapped host allocation, stream,
event and IPC mapping it made, in every configuration; and an allocation that fails inside an entry point makes it return
SERFSIM_E_NOMEM and leaves a handle that, once the call is repeated, computes what a fresh handle computes.

The shim counts the resources alive (emu_live_allocs) and makes the k-th next allocation fail (emu_fail_alloc_at).  The
failure sweeps arm k = 1, 2, ... until the call makes fewer than k allocations, so every allocation of the call fails once."""
import ctypes as C
import gc
import threading

import numpy as np
import pytest

import parity_lib as P
import wire_lib as W
from emu_lib import emu_sim, lib
from serf_b200 import scenarios
from serf_b200.sim import SerfsimError

NOMEM = -4
NAMES, PAYLOADS = [b"deploy", b"rollback", b"restart"], [b"v1", b"", b"now"]


@pytest.fixture(scope="module")
def L():
    L = W.bind_product(lib())
    L.emu_live_allocs.restype = C.c_long
    L.emu_fail_alloc_at.argtypes = [C.c_long]
    L.emu_fail_alloc_at(0)
    return L


def small():
    return scenarios.random_graph_leave(600, 8, 3, seed=2, slots=1)


def storm():
    return scenarios.user_event_storm(600, 8, 3, seed=3, n_events=3, spacing=2, churn=10)


def run(g, sc):
    g.run_until_converged(sc.max_ticks)


def baseline(L):
    """The resources alive before a measurement.  Handles that earlier tests of this process left in reference cycles are freed
    first: the cycle collector could otherwise free them in the middle of the measurement."""
    gc.collect()
    return L.emu_live_allocs()


# ---- part 1: every configuration releases what it allocated --------------------------------------------------------
def wire_all(g, sc):
    buf, off = g.wire_local_state_range()
    W.decode_batch(lib(), g, buf, off, sc.slots)
    g.wire_decode_events(buf, off)


def ranks(world, sc, timing, **cfg):
    """sc on `world` ranks, threads of this process, every handle closed before returning."""
    comm, errs = P.ThreadComm(world), []

    def rank(r):
        try:
            g = sc.build(emu_sim, rank=r, world_size=world, **cfg)
            g.set_tick_timing(timing)
            g.connect(*comm.hooks(r))
            run(g, sc)
            comm.bar.wait()                              # no rank closes its windows while another still reads them
            g.close()
        except BaseException as e:                       # noqa: BLE001 — surface it in the test thread
            errs.append(e)
            comm.bar.abort()
    th = [threading.Thread(target=rank, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(600)
    if errs:
        raise errs[0]


def single(sc, then=None, **cfg):
    g = sc.build(emu_sim, **cfg)
    if then:
        then(g, sc)
    else:
        run(g, sc)
    g.close()


def with_content(g, sc):
    g.set_user_event_content(NAMES, PAYLOADS)
    run(g, sc)
    wire_all(g, sc)


def results(g, sc):
    run(g, sc)
    for _ in range(6):                                   # more calls than the ring has buffers
        st, lt, lam = np.zeros(g.count, np.uint8), np.zeros(g.count, np.uint32), np.zeros(g.count, np.uint32)
        g.results_async(0, status=st, status_ltime=lt, lamport=lam)
        g.results_wait()


def topology_twice(g, sc):
    g.set_topology(sc.row_ptr, sc.col)
    run(g, sc)


def many_ops(g, sc):
    for node in range(1, 1100):                          # more operations than the first op table holds
        g.rejoin(node % sc.n, tick=node // sc.n)
    g.step(4)


def loopback():
    g = scenarios.random_graph_leave(4000, 12, 3, seed=2, slots=1).build(emu_sim, rank=0, world_size=4)
    g.connect_loopback()
    g.run_until_converged(400)
    g.close()


CASES = {
    "single_slot": lambda: single(small()),
    "multi_slot_carry": lambda: single(scenarios.random_graph_leave(600, 8, 3, seed=2, slots=3)),
    "push_pull": lambda: single(small(), push_pull_interval_ticks=5),
    "user_events_content_push_pull": lambda: single(storm(), with_content, push_pull_interval_ticks=5),
    "injectors": lambda: single(scenarios.byzantine_injectors(600, 8, 3, 0.05, seed=1)),
    "tick_timing": lambda: single(small(), lambda g, sc: (g.set_tick_timing(True), run(g, sc))),
    "results_async": lambda: single(small(), results),
    "records": lambda: single(small(), lambda g, sc: (run(g, sc), g.records(0))),
    "set_topology_twice": lambda: single(small(), topology_twice),
    "trace_growth": lambda: single(small(), lambda g, sc: g.step(1100)),
    "op_table_growth": lambda: single(small(), many_ops),
    "sharded_w2": lambda: ranks(2, storm(), True, push_pull_interval_ticks=5),
    "sharded_w3": lambda: ranks(3, storm(), True, push_pull_interval_ticks=5),
    "sharded_timed_w2": lambda: ranks(2, scenarios.random_graph_leave(3000, 8, 3, seed=2, slots=1), True),
    "loopback": loopback,
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_closed_handles_release_everything(L, case):
    base = baseline(L)
    CASES[case]()
    assert L.emu_live_allocs() == base


# ---- part 2: an allocation that fails leaves a usable handle --------------------------------------------------------
def rc_of(f):
    try:
        return 0, f()
    except SerfsimError as e:
        return e.code, None


def sweep(L, make, call, rest):
    """make() -> a handle ready for call(g) -> (rc, value); rest(g, value) -> the outputs the handle then computes.  For every
    allocation of call: it fails with SERFSIM_E_NOMEM, the repeated call succeeds, the outputs equal those of a handle whose
    call never failed, and every handle releases everything.  Returns the number of allocations the call makes."""
    base = baseline(L)
    g = make()
    rc, value = call(g)
    assert rc == 0, rc
    ref = rest(g, value)
    g.close()
    k = 1
    while True:
        g = make()
        L.emu_fail_alloc_at(k)
        try:
            rc, value = call(g)
        finally:
            L.emu_fail_alloc_at(0)
        if rc == 0:                                      # the call makes fewer than k allocations
            g.close()
            assert L.emu_live_allocs() == base
            return k - 1
        assert rc == NOMEM, (k, rc)
        rc, value = call(g)
        assert rc == 0, (k, rc)
        P.assert_same(rest(g, value), ref, with_hash=False, what=f"allocation {k} of the call failed")
        g.close()
        assert L.emu_live_allocs() == base, k
        k += 1


def outputs(sc, steps=None):
    def rest(g, value):
        out = P.outputs(g, sc, g.run_until_converged(sc.max_ticks) if steps is None else g.step(steps))
        if value is not None:
            out["value"] = list(value)
        return out
    return rest


def bare(sc, **cfg):
    def make():
        g = emu_sim(sc.n, sc.slots, **dict(sc.cfg, **cfg))
        g.set_topology(sc.row_ptr, sc.col)
        g.set_subjects(sc.subjects)
        return g
    return make


def then_schedule(sc, f):
    """f(g) as a sweep call that, once it succeeds, schedules sc's operations."""
    def call(g):
        rc, value = rc_of(lambda: f(g))
        if rc == 0:
            sc.schedule(g)
        return rc, value
    return call


@pytest.mark.parametrize("cfg", [dict(), dict(slots=3), dict(push_pull_interval_ticks=5),
                                 dict(world_size=2, push_pull_interval_ticks=5), dict(world_size=3, slots=2)],
                         ids=["single_slot", "multi_slot", "push_pull", "sharded_push_pull", "sharded_multi_slot"])
def test_create_fails_cleanly_at_every_allocation(L, cfg):
    """serfsim_create, including the push-pull snapshots (allocated by create so that a round never allocates mid-tick)."""
    cfg = dict(cfg)
    slots = cfg.pop("slots", 1)
    base = baseline(L)
    k = 1
    while True:
        L.emu_fail_alloc_at(k)
        try:
            rc, g = rc_of(lambda: emu_sim(600, slots, **cfg))
        finally:
            L.emu_fail_alloc_at(0)
        if rc == 0:
            g.close()
            break
        assert rc == NOMEM, (k, rc)
        assert L.emu_live_allocs() == base, k
        k += 1
    assert L.emu_live_allocs() == base
    assert k > 20


def test_set_user_events_sweep(L):
    sc = storm()
    call = then_schedule(sc, lambda g: g.set_user_events(sc.user_events))
    assert sweep(L, bare(sc, push_pull_interval_ticks=5), call, outputs(sc)) == 7


def test_set_user_event_content_sweep(L):
    sc = storm()
    make = lambda: sc.build(emu_sim)
    call = lambda g: rc_of(lambda: g.set_user_event_content(NAMES, PAYLOADS))
    rest = lambda g, _: dict(outputs(sc)(g, None), wire=list(g.wire_local_state_range()))      # the rings carry the content
    assert sweep(L, make, call, rest) == 1


def test_set_byzantine_sweep(L):
    sc = scenarios.byzantine_injectors(600, 8, 3, 0.05, seed=1)
    call = then_schedule(sc, lambda g: g.set_byzantine(sc.byzantine, sc.delta))
    assert sweep(L, bare(sc), call, outputs(sc)) == 3


def test_results_async_sweep(L):
    sc = small()

    def make():
        g = sc.build(emu_sim)
        run(g, sc)
        return g

    def call(g):
        st, lt, lam = np.zeros(g.count, np.uint8), np.zeros(g.count, np.uint32), np.zeros(g.count, np.uint32)
        rc, _ = rc_of(lambda: g.results_async(0, status=st, status_ltime=lt, lamport=lam))
        if rc == 0:
            g.results_wait()
        return rc, [st, lt, lam]
    assert sweep(L, make, call, outputs(sc, steps=0)) == 10          # copy stream and event, four buffers and their events


def test_trace_and_op_table_growth_sweep(L):
    """The first step of a handle sizes the op table (1024 operations) and a step past 1024 ticks grows the trace arrays: both
    before any tick of the call is launched."""
    sc = small()
    make = lambda: sc.build(emu_sim)
    call = lambda g: rc_of(lambda: g.step(1100))
    assert sweep(L, make, call, outputs(sc, steps=0)) == 6


def test_op_table_growth_sweep(L):
    sc = small()

    def make():
        g = sc.build(emu_sim)
        g.step(1)
        for node in range(1, 1100):
            g.rejoin(node % sc.n, tick=1 + node // sc.n)
        return g
    call = lambda g: rc_of(lambda: g.step(4))
    assert sweep(L, make, call, outputs(sc)) == 3


def wire_range(g, size):
    off, tot, out = np.zeros(g.count + 1, np.uint64), C.c_size_t(), np.zeros(size, np.uint8)
    rc = lib().serfsim_wire_local_state_range(g._h, 0, g.count, out.ctypes.data, out.size, off.ctypes.data, C.byref(tot))
    return rc, [out[:tot.value], off]


def test_wire_batches_sweep(L):
    sc = storm()

    def make():
        g = sc.build(emu_sim)
        g.set_user_event_content(NAMES, PAYLOADS)
        run(g, sc)
        return g
    g = make()
    buf, off = g.wire_local_state_range()
    g.close()
    rest = outputs(sc, steps=0)
    assert sweep(L, make, lambda g: wire_range(g, buf.size), rest) == 3
    assert sweep(L, make, lambda g: W.decode_batch(L, g, buf, off, sc.slots, check=False), rest) == 7

    def events(g):
        n = off.size - 1
        ev, seen, um = np.zeros(n, np.uint64), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        rc = lib().serfsim_wire_decode_events_batch(g._h, buf.ctypes.data, off.ctypes.data, n, ev.ctypes.data, seen.ctypes.data, um.ctypes.data)
        return rc, [ev, seen, um]
    assert sweep(L, make, events, rest) == 6
