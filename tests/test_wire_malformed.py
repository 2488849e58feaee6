"""The wire decoders on malformed and boundary bytes, on the CPU: the deterministic corpus of tests/wire_malformed_lib.py (and
random mutations of its seeds) through the product's host decoders, the oracle and the restatement — error class and decoded
values compared three ways, with the documented differences listed in that module — then through both batch kernels (host
build of tests/emu): alone and inside a batch of valid messages, the call must fail at the first bad index with the host
decoder's class, or decode every message as the host decoders do.  Also the offsets rule of the batch entry points
(include/serfsim.h).  The same corpus runs through the device kernels in tests/test_gpu_z_wire_malformed.py."""
import collections

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import ue_wire_ref as R
import wire_events_lib as WE
import wire_lib as W
import wire_malformed_lib as ML
from emu_lib import emu_sim, lib as emu_lib
from serf_b200 import scenarios
from serf_b200.sim import SerfsimError
from test_wire_events import content_of, set_content


@pytest.fixture(scope="module")
def P():
    return WE.bind(emu_lib())                    # the product's wire_codec.cu compiled for the host (no GPU here)


@pytest.fixture(scope="module")
def CASES():
    return ML.corpus()


def batch_sim(build):
    """A small run with 3 tracked user events (content table set, events fired): its own push-pull messages are the valid
    neighbours of the batch tests and match tracked events."""
    sc = scenarios.user_event_storm(400, 8, 3, seed=1, n_events=3, spacing=2)
    g = sc.build(build, trace=0)
    set_content(g, sc.user_events)
    g.step(12)
    names, pays = zip(*[content_of(c) for c in sc.user_events])
    table = (list(names), list(pays), [g.user_event_ltime(e) for e in range(len(names))])
    buf, off = g.wire_local_state_range(0, 6)
    valid = [bytes(buf[int(off[i]):int(off[i + 1])]) for i in range(6)]
    return g, table, valid


@pytest.fixture(scope="module")
def SIM():
    g, table, valid = batch_sim(emu_sim)
    yield g, table, valid
    g.close()


# ---- the corpus itself ----
def test_seeds_are_the_encoders_bytes():
    for name, (fn, args) in ML.SEEDS.items():
        b = ML.ser(ML.seed_tree(name))
        if fn is ML.t_join:
            assert b == W.o_encode_intent(W.JOIN, *args)
        elif fn is ML.t_leave:
            assert b == W.o_encode_intent(W.LEAVE, *args)
        elif fn is ML.t_push_pull:
            assert b == R.push_pull(*args)
        else:
            assert b == R.user_event_message(*args)


def test_corpus_covers_every_edge(CASES):
    assert len(CASES) > 3000
    by = collections.defaultdict(set)
    for c in CASES:
        by[(c.seed, c.family)].add(c.attr)
    for name in ML.SEEDS:
        tree = ML.seed_tree(name)
        n = len(ML.ser(tree))
        assert by[(name, "truncate")] == {(k,) for k in range(n)}                    # every byte offset
        for path, f in ML.walk(tree):
            w = f.tag & 7
            if w == ML.VARINT:                                                       # every varint: lengths 1-10, 10th / 11th byte, overlong
                got = {a[1:] for a in by[(name, "varint")] if a[0] == path}
                assert {("len", L, m) for L in range(1, 11) for m in ("min", "max")} <= got
                assert {("tenth", x) for x in (1, 2, 0x7F, 0x81)} | {("eleven", "ff"), ("overlong", "80 00"), ("overlong", "ff 80 00")} <= got
            if w == ML.LEN:                                                          # every length prefix: rem, rem + 1, 2^32 - 1, 2^32, 2^64 - 1
                assert {a[1] for a in by[(name, "len")] if a[0] == path} == set(ML.LEN_FORMS)
            assert {a[1] for a in by[(name, "retype")] if a[0] == path} == set(range(8)) - {w}
            assert (path,) in by[(name, "duplicate")] and (path,) in by[(name, "remove")] and (path,) in by[(name, "duplicate_cut")]
        for cpath, cont in ML.containers(tree):                                      # unknown fields of every wire type at every boundary
            assert {(cpath, i, w) for i in range(len(cont) + 1) for w in range(8)} <= by[(name, "unknown")]
            assert {(cpath, w) for w in range(5)} <= by[(name, "unknown_cut")]
        assert {a[0] for a in by[(name, "two")]} == set(ML.SEEDS)                    # two messages, every pair, both orders


# ---- pinned classes at the varint and length boundaries ----
def join_with_ltime(raw):
    body = bytes([0x09]) + raw + bytes([0x11, 9])
    return bytes([0x12, len(body)]) + body


@pytest.mark.parametrize("raw,want", [
    (b"\xff" * 9 + b"\x01", ("ok", 2**64 - 1)),                                     # 10th byte 01: bit 63
    (b"\x80" * 9 + b"\x01", ("ok", 2**63)),
    (b"\xff" * 9 + b"\x02", ("err", "varint")),                                      # 10th byte > 1: more than 64 bits
    (b"\xff" * 9 + b"\x7f", ("err", "varint")),
    (b"\xff" * 9 + b"\x81", ("err", "varint")),
    (b"\x80" * 10 + b"\x00", ("err", "varint")),                                     # 11 bytes
    (b"\x80\x00", ("ok", 0)),                                                        # overlong, zero-padded: accepted (UNPINNED)
    (b"\xff\x80\x00", ("ok", 127)),
    (b"\x80" * 9 + b"\x00", ("ok", 0)),
])
def test_varint_boundaries_in_every_decoder(P, raw, want):
    b = join_with_ltime(raw)
    got = ML.product(P, b)["intent"]
    assert (got[0], got[1][1] if got[0] == "ok" else got[1]) == want
    assert ML.disagreements(P, b) == []


@pytest.mark.parametrize("declared,want", [("rem", "ok"), ("rem+1", "truncated"), (2**32 - 1, "truncated"), (2**32, "truncated"), (2**64 - 1, "truncated")])
def test_length_prefix_boundaries_in_every_decoder(P, declared, want):
    def prefix(rem):                                                                 # declared length against the rem bytes left
        return R.varint(rem if declared == "rem" else rem + 1 if declared == "rem+1" else declared)
    # an unknown length-delimited field as the last field of a Join, a UserEventMessage name, and the envelope itself
    body = bytes([0x09, 5, 0x11, 9, 0x7A]) + prefix(3) + b"abc"
    uem = bytes([0x09, 5, 0x1A]) + prefix(2) + b"nm"
    uem_ok = bytes([0x09, 5, 0x1A, 2]) + b"nm"
    for m, k in ((bytes([0x12, len(body)]) + body, "intent"), (bytes([0x22, len(uem)]) + uem, "uem"), (bytes([0x22]) + prefix(len(uem_ok)) + uem_ok, "uem")):
        got = ML.product(P, m)[k]
        assert (got[0] if want == "ok" else got[1]) == want, m.hex()
        assert ML.disagreements(P, m) == []


def test_unknown_wire_types(P):
    base = ML.seed_tree("join")
    for w, want in enumerate(["ok"] * 5 + ["wire_type"] * 3):
        b = ML.ser(ML.inserted(base, (0,), 1, ML.F(ML.UNKNOWN_TAG | w, raw=ML.UNKNOWN[w])))
        got = ML.product(P, b)["intent"]
        assert (got[0] if want == "ok" else got[1]) == want, w
        if w < 5:                                                                    # cut short as the last field: truncated
            b = ML.ser(ML.inserted(base, (0,), 2, ML.F(ML.UNKNOWN_TAG | w, raw=ML.UNKNOWN_CUT[w])))
            assert ML.product(P, b)["intent"] == ("err", "truncated"), w


# ---- three decoders, one corpus ----
def test_three_decoders_agree_on_the_corpus(P, CASES):
    bad, classes = [], collections.Counter()
    for c in CASES:
        d = ML.disagreements(P, c.data)
        if d:
            bad.append((c, d))
        for k, v in ML.product(P, c.data).items():
            classes[(k, v[0] if v[0] == "ok" else v[1])] += 1
    assert not bad, (len(bad), bad[:5])
    # the corpus reaches every error class of every decoder, and accepts a good share of its inputs
    for k in ("intent", "push_pull", "ring", "uem"):
        for cls in ("ok", "truncated", "varint", "duplicate", "missing", "wire_type", "type"):
            assert classes[(k, cls)] > 0, (k, cls)
    assert classes[("ring", "ok")] > 300 and classes[("intent", "ok")] > 200 and classes[("uem", "ok")] > 100


MUTATION = st.tuples(st.sampled_from(["truncate", "replace", "insert", "flip"]), st.integers(0, 2**16), st.integers(0, 255))


@settings(max_examples=3000, deadline=None)
@given(st.sampled_from(sorted(ML.SEEDS)), st.lists(MUTATION, min_size=1, max_size=4))
def test_random_mutations_three_decoders_agree(P, seed, muts):
    b = bytearray(ML.ser(ML.seed_tree(seed)))
    for op, pos, v in muts:
        i = pos % (len(b) + 1)
        if op == "truncate":
            del b[i:]
        elif op == "insert":
            b.insert(i, v)
        elif b:
            i %= len(b)
            b[i] = v if op == "replace" else b[i] ^ 0x80                             # flip: the continuation bit
    assert ML.disagreements(P, bytes(b)) == []


@pytest.mark.parametrize("cap", [1, 3, 16])
def test_capacity_exact_and_one_more(P, cap):
    for n_status, n_left in ((cap, cap), (cap + 1, cap), (cap, cap + 1)):
        b, status, _ = ML.capacity_message(n_status, n_left, [])
        over = n_status > cap or n_left > cap
        got = ML.p_decode_push_pull(P, b, cap=cap, left_cap=cap)
        assert (got[0] != 0) == over
        if over:
            assert ML.product_class(P.serfsim_last_error()) == "capacity"
        else:
            assert got[1][1] == status
        rc, _ = W.o_decode_push_pull(b, cap=cap)
        assert rc == (-6 if over else 0)
    # ring entries and events of the events decoder
    for ring_sizes, ring_cap, ev_cap in (([1] * cap, cap, cap), ([1] * (cap + 1), cap, cap + 1), ([cap], 1, cap), ([cap + 1], 1, cap)):
        b, _, ring = ML.capacity_message(0, 0, ring_sizes)
        over = len(ring) > ring_cap or sum(len(e) for _, e in ring) > ev_cap
        rc, v = WE.decode_push_pull(P, b, cap=0, ring_cap=ring_cap, ev_cap=ev_cap)
        assert (rc != 0) == over, (ring_sizes, ring_cap, ev_cap)
        if over:
            assert ML.product_class(P.serfsim_last_error()) == "capacity"
        else:
            assert v[4] == ring


# ---- the batch kernels (host build) ----
def test_batch_kernels_on_the_corpus(P, SIM, CASES):
    g, table, valid = SIM
    fails = collections.Counter()
    for i, c in enumerate(CASES):
        ML.check_in_batches(P, g, table, 3, c.data, valid[:4], i % 5)
        fails[ML.expect_decode_batch(P, c.data, 3)[0]] += 1
    assert fails["err"] > 1000 and fails["ok"] > 100


def test_batch_capacity_status_cap_and_16_left_entries(P, SIM):
    g, table, valid = SIM
    for n_status, n_left, want in ((3, 16, "ok"), (4, 0, "capacity"), (0, 17, "capacity")):
        b, _, _ = ML.capacity_message(n_status, n_left, [])
        assert ML.expect_decode_batch(P, b, 3)[0 if want == "ok" else 1] == want
        ML.check_in_batches(P, g, table, 3, b, valid, 2)


def test_batch_neighbour_cannot_complete_a_truncated_message(P, SIM):
    """Message k's envelope claims more bytes than its slice; the next message's bytes would complete it.  It must be
    truncated, not decoded from its neighbour's bytes."""
    g, table, valid = SIM
    for cut in (1, 3, len(valid[1]) - 2):
        msgs = [valid[0], valid[1][:-cut], valid[1][-cut:] + valid[2], valid[3]]
        assert bytes(b"".join(msgs[1:3])) == valid[1] + valid[2]
        assert ML.run_decode_batch(P, g, msgs, 3) == ("err", 1, "truncated")
        assert ML.run_events_batch(g, msgs) == ("err", 1, "truncated")


def random_messages(rng, table, n):
    names, pays, lts = table
    out = []
    for _ in range(n):
        status = [(int(rng.integers(0, 2**63)), int(rng.integers(0, 2**40))) for _ in range(rng.integers(0, 4))]
        left = [int(x) for x in rng.integers(0, 2**20, rng.integers(0, 3))]
        ring = []
        for _ in range(rng.integers(0, 3)):
            if rng.random() < 0.5:                                                   # a tracked event at its ltime
                e = int(rng.integers(0, len(names)))
                ring.append((lts[e], [(names[e], pays[e])]))
            else:
                ring.append((int(rng.integers(0, 2**32)), [(bytes(rng.integers(0, 256, rng.integers(0, 40), dtype=np.uint8)), b"p") for _ in range(rng.integers(0, 3))]))
        out.append(R.push_pull(int(rng.integers(0, 2**63)), status, left, int(rng.integers(0, 2**33)), ring, int(rng.integers(0, 9))))
    return out


def test_batch_edges(P, SIM):
    g, table, valid = SIM
    assert ML.run_decode_batch(P, g, [], 3) == ("ok", [])                            # n = 0
    assert ML.run_events_batch(g, []) == ("ok", [])
    for msgs, k in (([b""], 0), ([valid[0], b"", valid[1]], 1)):                      # a zero-length message: no message in it
        assert ML.run_decode_batch(P, g, msgs, 3) == ("err", k, "missing")
        assert ML.run_events_batch(g, msgs) == ("err", k, "missing")
    msgs = random_messages(np.random.default_rng(7), table, 3000)                    # thousands of messages of random sizes
    sizes = [len(m) for m in msgs]
    assert min(sizes) < 20 and max(sizes) > 150
    assert ML.run_decode_batch(P, g, msgs, 3) == ("ok", [ML.expect_decode_batch(P, m, 3)[1] for m in msgs])
    want = [ML.expect_events_batch(P, m, table)[1] for m in msgs]
    assert ML.run_events_batch(g, msgs) == ("ok", want)
    assert sum(1 for w in want if w[1]) > 1000                                      # tracked events matched


def test_batch_offsets_are_validated(P, SIM):
    g, table, valid = SIM
    buf, off = ML.pack(valid[:4])
    n = off.size - 1
    outs = [np.zeros(n * 4, np.uint64) for _ in range(3)] + [np.zeros(n, np.uint32)]
    ev, seen, um = np.zeros(n, np.uint64), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    for k in range(n):                                                               # offsets[k] > offsets[k + 1]: rejected, index named
        bad = off.copy()
        bad[k] = bad[k + 1] + 1
        assert P.serfsim_wire_decode_batch(g._h, buf.ctypes.data, bad.ctypes.data, n, 4, *[o.ctypes.data for o in outs]) == -1
        assert f"offsets[{k}] > offsets[{k + 1}]".encode() in P.serfsim_last_error()
        assert P.serfsim_wire_decode_events_batch(g._h, buf.ctypes.data, bad.ctypes.data, n, ev.ctypes.data, seen.ctypes.data, um.ctypes.data) == -1
        assert f"offsets[{k}] > offsets[{k + 1}]".encode() in P.serfsim_last_error()
        with pytest.raises(SerfsimError, match=rf"offsets\[{k}\] > offsets\[{k + 1}\]"):
            g.wire_decode_events(buf, bad)
    # the example of a message longer than the buffer: [0, 116, 32] over 32 bytes
    short = np.frombuffer(valid[0][:32].ljust(32, b"\0"), np.uint8)
    bad = np.array([0, 116, 32], np.uint64)
    assert P.serfsim_wire_decode_batch(g._h, short.ctypes.data, bad.ctypes.data, 2, 4, *[o.ctypes.data for o in outs]) == -1
    assert b"offsets[1] > offsets[2]" in P.serfsim_last_error()
    # offsets[n] past the end of the buffer, and no offsets at all: rejected before the C call
    past = off.copy()
    past[-1] += 1
    for call in (lambda o: g.wire_decode_events(buf, o), lambda o: W.decode_batch(P, g, buf, o, 4)):
        with pytest.raises(ValueError, match="past the end"):
            call(past)
        with pytest.raises(ValueError, match="n \\+ 1 entries"):
            call(np.zeros(0, np.uint64))
    assert ML.run_decode_batch(P, g, valid[:4], 4)[0] == "ok"                         # and the good offsets still decode
