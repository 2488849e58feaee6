"""User events on the wire, on the CPU: UserEventMessage and PushPull with the event ring (tests/ue_wire_ref.py restates them
independently) against hand-derived bytes and the round-trip property of types/tests.rs:8-25, the product's host codec against
the restatement byte for byte, every decode error path, the envelope cases that change with the user-event message byte,
the content table's rejections, and the batch kernels (host build of tests/emu) against rings taken from the ORACLE's run.
Byte-level interop with a real serf node stays UNPINNED: memberlist_core::proto is not in the reference tree (wire.cuh)."""
import ctypes as C
import threading

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import ue_wire_ref as R
import wire_events_lib as WE
import wire_lib as W
from emu_lib import emu_sim, lib as emu_lib
from oracle_lib import oracle_sim
from serf_b200 import scenarios
from serf_b200.sim import SerfsimError

U64 = st.integers(min_value=0, max_value=2**64 - 1)
SMALL = st.one_of(st.integers(0, 300), U64)
BLOB = st.binary(max_size=200)
EVENT = st.tuples(BLOB, BLOB)
RING = st.lists(st.tuples(SMALL, st.lists(EVENT, max_size=3)), max_size=4)


@pytest.fixture(scope="module")
def P():
    return WE.bind(emu_lib())                    # the product's wire_codec.cu compiled for the host (no GPU here)


def test_hand_derived_bytes(P):
    # The PushPull of the reference's delegate_merge_remote_state KAT (serf/base/tests/serf/delegate.rs:117-180) with u64 ids
    # (test = 7, foo = 8): its one events entry UserEvents{45, [UserEvent{"test", ""}]} is [0x2A = 5<<3|2][10][0x09 45]
    # [0x12 = 2<<3|2][6][UserEvent: 0x0A = 1<<3|2, 4, "test"] — the empty payload is not written (user_event.rs:122-130).
    events_field = bytes([0x2A, 0x0A, 0x09, 0x2D, 0x12, 0x06, 0x0A, 0x04, 0x74, 0x65, 0x73, 0x74])
    head = bytes([0x09, 42, 0x12, 4, 0x09, 7, 0x11, 20, 0x12, 4, 0x09, 8, 0x11, 15, 0x19, 8, 0x21, 50])
    body = head + events_field + bytes([0x31, 100])
    want = bytes([0x1A, len(body)]) + body
    args = (42, [(7, 20), (8, 15)], [8], 50, [(45, [(b"test", b"")])], 100)
    assert R.push_pull(*args) == want
    assert WE.encode_push_pull(P, *args) == want
    assert WE.decode_push_pull(P, want) == (0, args)
    # UserEventMessage{ltime 5, name "foo", payload empty, cc}: message byte 4<<3|2 = 0x22; ltime 0x09; cc 2<<3|0 = 0x10 then 1;
    # name 3<<3|2 = 0x1A; no payload field (message.rs:224-271)
    uem = bytes([0x22, 9, 0x09, 5, 0x10, 1, 0x1A, 3, 0x66, 0x6F, 0x6F])
    assert R.user_event_message(5, b"foo", b"", True) == uem
    assert WE.encode_user_event(P, 5, b"foo", b"", True) == uem
    assert WE.decode_user_event(P, uem) == (0, (5, b"foo", b"", True))


def test_restatement_agrees_with_the_oracle_without_events():
    for args in [(42, [(7, 20)], [7], 50, 100), (2**40, [(1, 2), (3, 2**33)], [], 1, 1), (0, [], [], 0, 0)]:
        lt, status, left, ev, q = args
        assert R.push_pull(lt, status, left, ev, [], q) == W.o_encode_push_pull(*args)


@settings(max_examples=300, deadline=None)
@given(SMALL, BLOB, BLOB, st.booleans())
def test_user_event_round_trip_and_product_equals_restatement(P, ltime, name, payload, cc):
    b = R.user_event_message(ltime, name, payload, cc)
    assert R.d_user_event_message(b) == (ltime, name, payload, cc)                  # data_round_trip, types/tests.rs:8-25
    assert WE.encode_user_event(P, ltime, name, payload, cc) == b
    assert WE.decode_user_event(P, b) == (0, (ltime, name, payload, cc))
    t = C.c_uint32()
    assert P.serfsim_wire_message_type(W._buf(b), len(b), C.byref(t)) == 0 and t.value == WE.USER_EVENT


@settings(max_examples=200, deadline=None)
@given(SMALL, st.lists(st.tuples(SMALL, SMALL), max_size=6, unique_by=lambda kv: kv[0]), st.lists(SMALL, max_size=4, unique=True), SMALL, RING, SMALL)
def test_push_pull_with_events_round_trip_and_product_equals_restatement(P, ltime, status, left, ev, ring, q):
    b = R.push_pull(ltime, status, left, ev, ring, q)
    assert R.d_push_pull(b) == (ltime, status, left, ev, ring, q)
    assert WE.encode_push_pull(P, ltime, status, left, ev, ring, q) == b
    assert WE.decode_push_pull(P, b) == (0, (ltime, status, left, ev, ring, q))
    # the membership decoder still counts and skips the entries
    assert W.p_decode_push_pull(P, b) == (0, (ltime, status, left, ev, q, len(ring)))


def _fails_both(P, b, which):
    with pytest.raises(R.WireError):
        (R.d_user_event_message if which == "uem" else R.d_push_pull)(b)
    rc = (WE.decode_user_event if which == "uem" else WE.decode_push_pull)(P, b)[0]
    assert rc != 0


def test_user_event_decode_errors_and_unknown_fields(P):
    uem = R.user_event_message(300, b"name", b"pay", True)
    _fails_both(P, uem[:-1], "uem")                                                  # truncated
    _fails_both(P, bytes([0x22, 4, 0x09, 5, 0x09, 6]), "uem")                        # ltime twice
    _fails_both(P, bytes([0x22, 6, 0x09, 5, 0x10, 1, 0x10, 0]), "uem")              # cc twice
    _fails_both(P, bytes([0x22, 8, 0x09, 5, 0x1A, 1, 0x61, 0x1A, 1, 0x62]), "uem")   # name twice
    _fails_both(P, bytes([0x22, 8, 0x09, 5, 0x22, 1, 0x61, 0x22, 1, 0x62]), "uem")   # payload twice
    _fails_both(P, bytes([0x22, 3, 0x1A, 1, 0x61]), "uem")                           # ltime missing (message.rs:181)
    # unknown fields (tag 7 varint, tag 6 length-delimited) are skipped; name / payload default to empty, cc to false
    ext = bytes([0x22, 9, 0x39, 0x7F, 0x09, 5, 0x32, 3, 1, 2, 3])
    assert R.d_user_event_message(ext) == (5, b"", b"", False)
    assert WE.decode_user_event(P, ext) == (0, (5, b"", b"", False))
    assert WE.decode_user_event(P, W.o_encode_intent(W.JOIN, 5, 9))[0] != 0         # not a user-event message


def test_push_pull_events_decode_errors_and_capacity(P):
    def pp(entry):                                                                   # a PushPull whose one events entry is `entry`
        body = bytes([0x09, 1, 0x21, 2]) + R.ld(0x2A, entry) + bytes([0x31, 1])
        return bytes([0x1A, len(body)]) + body
    ok = pp(R.user_events(45, [(b"a", b"b")]))
    assert WE.decode_push_pull(P, ok) == (0, (1, [], [], 2, [(45, [(b"a", b"b")])], 1))
    _fails_both(P, pp(bytes([0x12, 2, 0x0A, 0])), "pp")                              # UserEvents without ltime
    _fails_both(P, pp(bytes([0x09, 1, 0x09, 2])), "pp")                              # UserEvents ltime twice
    _fails_both(P, pp(bytes([0x09, 1, 0x12, 6, 0x0A, 1, 0x61, 0x0A, 1, 0x62])), "pp")   # UserEvent name twice
    _fails_both(P, pp(bytes([0x09, 1, 0x12, 6, 0x12, 1, 0x61, 0x12, 1, 0x62])), "pp")   # UserEvent payload twice
    _fails_both(P, pp(bytes([0x09, 1, 0x12, 5, 0x0A, 4, 0x61])), "pp")              # UserEvent truncated inside its entry
    _fails_both(P, ok[:-3], "pp")                                                    # truncated message
    # unknown fields inside UserEvents and UserEvent are skipped
    ext = pp(bytes([0x39, 3, 0x09, 45, 0x12, 7, 0x39, 1, 0x0A, 1, 0x61, 0x18, 0]))
    assert R.d_push_pull(ext)[4] == [(45, [(b"a", b"")])]
    assert WE.decode_push_pull(P, ext)[1][4] == [(45, [(b"a", b"")])]
    # caller-given capacities: ring entries and the event pool
    two = R.push_pull(1, [], [], 2, [(3, [(b"x", b"")]), (4, [(b"y", b""), (b"z", b"")])], 1)
    assert WE.decode_push_pull(P, two, ring_cap=2, ev_cap=3)[0] == 0
    assert WE.decode_push_pull(P, two, ring_cap=1, ev_cap=3)[0] != 0
    assert WE.decode_push_pull(P, two, ring_cap=2, ev_cap=2)[0] != 0
    assert WE.decode_push_pull(P, two, cap=0)[0] == 0                               # no status / left entries to store
    m = WE.UserEventMsg(2**40, None, 0, None, 0, 1, 0)
    n, out = C.c_size_t(), (C.c_uint8 * 4)()
    assert P.serfsim_wire_encode_user_event(C.byref(m), out, 4, C.byref(n)) != 0 and n.value == len(R.user_event_message(2**40, b"", b"", True))


def test_envelope_with_a_user_event_message(P):
    uem = R.user_event_message(7, b"deploy", b"v2", False)
    t = C.c_uint32()
    assert P.serfsim_wire_message_type(W._buf(uem), len(uem), C.byref(t)) == 0 and t.value == WE.USER_EVENT
    for b in (uem, bytes([0x39, 1]) + uem):                                          # alone, or after an unknown field
        rc, _ = W.p_decode_intent(P, b)
        assert rc != 0 and b"not a message of the requested type" in P.serfsim_last_error()
        rc, _ = W.p_decode_push_pull(P, b)
        assert rc != 0 and b"not a message of the requested type" in P.serfsim_last_error()
    for other in (W.o_encode_intent(W.JOIN, 5, 9), W.o_encode_push_pull(42, [(7, 20)], [7], 50, 100)):
        for b in (uem + other, other + uem):                                         # two messages: duplicate field (message.rs:568-576)
            assert W.p_decode_intent(P, b)[0] != 0 and b"duplicate field" in P.serfsim_last_error()
            assert W.p_decode_push_pull(P, b)[0] != 0 and b"duplicate field" in P.serfsim_last_error()
            assert P.serfsim_wire_message_type(W._buf(b), len(b), C.byref(t)) != 0


# ---- the simulator's rings ----
def content_of(cid):
    """Deterministic bytes for a content id: equal ids, equal bytes."""
    cid = int(cid)
    return f"event-{cid}".encode(), bytes((cid * 31 + k) & 0xFF for k in range((cid * 7) % 41))


def set_content(sim, ids):
    names, pays = zip(*[content_of(c) for c in ids])
    sim.set_user_event_content(list(names), list(pays))


def canonical(seen, ids, lt):
    """Tracked events with equal content and equal ltime are one event on the wire: map each to the lowest such index."""
    out = np.zeros_like(seen)
    for e in range(len(ids)):
        lo = min(j for j in range(len(ids)) if ids[j] == ids[e] and lt[j] == lt[e])
        out |= ((seen >> e) & 1) << lo
    return out


def oracle_view(o, sc):
    E = len(sc.user_events)
    rec = o.user_event_records()
    return dict(status=[o.member_status(s) for s in range(sc.slots)], ltime=[o.status_ltime(s) for s in range(sc.slots)], clock=o.lamport_time(),
                event_time=o.event_time(), seen=rec["seen"].astype(np.uint32),
                ue_ltime=[o.user_event_ltime(e) for e in range(E)])


def expected(view, sc, v):
    ltime, status, left = W.expected_local_state(view, v, sc.subjects)
    contents = [content_of(c) for c in sc.user_events]
    ring = R.ring_of(int(view["seen"][v]), view["ue_ltime"], contents)
    return R.push_pull(ltime, status, left, int(view["event_time"][v]), ring, 1)


def check_batches(g, o, sc, ticks_list, sample=23):
    E = len(sc.user_events)
    for ticks in ticks_list:
        o.step(ticks); g.step(ticks)
        view = oracle_view(o, sc)
        buf, off = g.wire_local_state_range()
        assert off[0] == 0 and off.size == sc.n + 1
        nodes = list(range(0, sc.n, sample)) + [int(x) for x in np.flatnonzero(view["seen"])[:50]]
        for v in nodes:
            assert bytes(buf[int(off[v]):int(off[v + 1])]) == expected(view, sc, v), (ticks, v)
        # the range API is the matching slice of the full batch
        for first, count in ((0, 1), (17, 333), (sc.n - 5, 5), (sc.n, 0)):
            rb, ro = g.wire_local_state_range(first, count)
            assert (ro == off[first:first + count + 1] - off[first]).all()
            assert bytes(rb) == bytes(buf[int(off[first]):int(off[first + count])])
        # and back: decode_events_batch gives user_event_seen / event_time for every node
        ev, seen, um = g.wire_decode_events(buf, off)
        assert (ev == g.event_time()).all() and (um == 0).all()
        mask = np.zeros(sc.n, np.uint32)
        for e in range(E):
            mask |= g.user_event_seen(e).astype(np.uint32) << e
        lt = [g.user_event_ltime(e) for e in range(E)]
        assert (canonical(seen, sc.user_events, lt) == canonical(mask, sc.user_events, lt)).all()
    return buf, off


@pytest.mark.parametrize("case", ["alias_churn", "push_pull_rounds"])
def test_local_state_with_rings_equals_oracle_rings(case):
    if case == "alias_churn":
        sc = scenarios.user_event_storm(2500, 12, 3, seed=5, n_events=4, spacing=2, alias=True, churn=40)
        cfg = {}
    else:
        sc = scenarios.user_event_storm(2000, 8, 2, seed=6, n_events=5, spacing=2, churn=30, with_leave=True)
        cfg = dict(push_pull_interval_ticks=7, retransmit_mult=1)
    o = sc.build(oracle_sim, trace=0, **cfg)
    g = sc.build(emu_sim, trace=0, **cfg)
    set_content(g, sc.user_events)
    check_batches(g, o, sc, (0, 3, 9, 40))


def test_content_table_rules():
    sc = scenarios.user_event_storm(400, 8, 3, seed=1, n_events=3, spacing=2)
    g = sc.build(emu_sim, trace=0)
    ids = sc.user_events
    plain, plain_off = g.wire_local_state_range()
    with pytest.raises(SerfsimError):
        g.set_user_event_content([b"a"], [b""])                                      # n differs from set_user_events
    names, pays = [content_of(c)[0] for c in ids], [content_of(c)[1] for c in ids]
    with pytest.raises(SerfsimError, match="name \\+ payload"):
        g.set_user_event_content([b"x" * 300] + names[1:], [b"y" * 213] + pays[1:])
    with pytest.raises(SerfsimError, match="encoded UserEventMessage"):
        g.set_user_event_content([b"x" * 250] + names[1:], [b"y" * 255] + pays[1:])  # 505 bytes, 520 encoded
    with pytest.raises(SerfsimError, match="equal content ids but different bytes"):
        g2 = scenarios.user_event_storm(400, 8, 3, seed=1, n_events=3, alias=True).build(emu_sim, trace=0)
        g2.set_user_event_content([b"a", b"b", b"c"], [b"", b"", b""])
    with pytest.raises(SerfsimError, match="different content ids but equal bytes"):
        g.set_user_event_content([b"a", b"a", b"c"], [b"p", b"p", b""])
    g.set_user_event_content([b"x" * 250] + names[1:], [b"y" * 247] + pays[1:])      # 497 bytes, 512 encoded: accepted
    set_content(g, ids)
    g.step(12)
    with_ring, _ = g.wire_local_state_range()
    g.reset(sc.cfg.get("seed", 1)); sc.schedule(g); g.step(12)
    assert bytes(g.wire_local_state_range()[0]) == bytes(with_ring)                  # reset keeps the table
    g.close()
    # without a content table the output is what it was: no events attached
    g = sc.build(emu_sim, trace=0)
    g.step(12)
    buf, off = g.wire_local_state_range()
    o = sc.build(oracle_sim, trace=0); o.step(12)
    view = oracle_view(o, sc)
    for v in range(0, sc.n, 7):
        ltime, status, left = W.expected_local_state(view, v, sc.subjects)
        assert bytes(buf[int(off[v]):int(off[v + 1])]) == R.push_pull(ltime, status, left, int(view["event_time"][v]), [], 1)
    set_content(g, ids)
    assert len(g.wire_local_state_range()[0]) > len(buf)
    g.reset(1)
    g.set_user_events(ids)                                                           # a new event table drops the content
    with pytest.raises(SerfsimError):
        g.wire_decode_events(buf, off)
    assert plain.size and plain_off[-1] == plain.size


def test_sharded_batches_concatenate_to_the_single_batch():
    from parity_lib import ThreadComm
    sc = scenarios.user_event_storm(1800, 8, 3, seed=3, n_events=4, spacing=2, churn=20)
    ticks = 25
    g1 = sc.build(emu_sim, trace=0)
    set_content(g1, sc.user_events)
    g1.step(ticks)
    want, _ = g1.wire_local_state_range()
    world, comm, out, errs = 2, ThreadComm(2), [None, None], []

    def worker(rank):
        try:
            g = sc.build(emu_sim, rank=rank, world_size=world, trace=0)
            set_content(g, sc.user_events)
            g.connect(*comm.hooks(rank))
            g.step(ticks)
            out[rank] = bytes(g.wire_local_state_range()[0])
            comm.bar.wait()
        except BaseException as e:                                                   # noqa: BLE001 — surface it in the main thread
            errs.append(e)
            comm.bar.abort()
    th = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(600)
    if errs:
        raise errs[0]
    assert out[0] + out[1] == bytes(want)
