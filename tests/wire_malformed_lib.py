"""Malformed and boundary bytes for serf's wire decoders — test infrastructure shared by tests/test_wire_malformed.py (the host
codec and the host build of the batch kernels) and tests/test_gpu_z_wire_malformed.py (the batch kernels on the device).

The corpus is generated deterministically from seven seed messages held as field trees (`F`), so that every varint, every
length prefix and every field boundary can be rewritten on its own and the enclosing lengths re-derived.  Each input is then
given to three independent decoders and their outcomes compared — error class AND decoded values:
  * the product: serf_b200/csrc/wire.cuh + wire_codec.cu (host entry points; the class is read back from serfsim_last_error);
  * the oracle: oracle/wire_oracle.cpp (-1 for truncated / varint / wire-type errors: a coarse class "malformed");
  * the restatement: tests/ue_wire_ref.py (WireError strings, one to one with the product's classes).

Documented differences (every other disagreement is a finding):
  * the oracle's envelope does not know the UserEventMessage byte 0x22 and skips it as an unknown field, so an input with
    0x22 at the top level of its envelope stream is checked against the restatement only;
  * the membership decoders (product serfsim_wire_decode_push_pull, oracle) count and skip `events` entries without parsing
    them, the restatement and serfsim_wire_decode_push_pull_events parse them: membership is compared with the oracle, the
    ring with the restatement;
  * the restatement has no capacities; the capacity cases are checked against counts instead;
  * serfsim_wire_decode_batch decodes left_members into a MAX_SLOTS (16) array it does not return: a message with 17 or
    more left entries fails there with "output capacity too small", as the host decoder does with a left capacity of 16.
Overlong (zero-padded) varints such as 80 00 and FF 80 00 are accepted, with their value, by all three decoders.  Whether
memberlist_core::proto's varint decoder does the same is not pinned: that crate is not in the reference tree (wire.cuh)."""
import copy
import ctypes as C
import re

import numpy as np

import ue_wire_ref as R
import wire_events_lib as WE
import wire_lib as W

BYTE, VARINT, LEN = 0, 1, 2
MAX_SLOTS = 16                                   # record.cuh: the left_members array of the decode kernel
BIG = 4096                                       # capacities that no corpus input reaches


# ---- field trees ----
class F:
    """One field: tag byte and value — int (Byte / Varint), bytes (a length-delimited blob) or a list of F (a nested message,
    length-delimited).  raw: the bytes after the tag byte, as given (a rewritten varint, an unknown field's value).
    prefix(n, rem): the length prefix of a length-delimited field with n value bytes and rem bytes left in its parent after
    the prefix (None: varint(n))."""
    __slots__ = ("tag", "val", "raw", "prefix")

    def __init__(self, tag, val=None, raw=None, prefix=None):
        self.tag, self.val, self.raw, self.prefix = tag, val, raw, prefix


def ser(fields):
    out = b""
    for f in reversed(fields):                   # back to front: a prefix may depend on the bytes after its field
        out = enc(f, len(out)) + out
    return out


def enc(f, after):
    if f.raw is not None:
        return bytes([f.tag]) + f.raw
    w = f.tag & 7
    if w == BYTE:
        return bytes([f.tag, f.val])
    if w == VARINT:
        return bytes([f.tag]) + R.varint(f.val)
    v = ser(f.val) if isinstance(f.val, list) else bytes(f.val)
    return bytes([f.tag]) + (f.prefix(len(v), len(v) + after) if f.prefix else R.varint(len(v))) + v


def walk(tree, path=()):
    """(path, field) for every field, depth first; path = indices through nested lists."""
    for i, f in enumerate(tree):
        yield path + (i,), f
        if isinstance(f.val, list):
            yield from walk(f.val, path + (i,))


def containers(tree, path=()):
    """(path, list) for the envelope stream and every nested message."""
    yield path, tree
    for i, f in enumerate(tree):
        if isinstance(f.val, list):
            yield from containers(f.val, path + (i,))


def _parent(tree, path):
    for i in path:
        tree = tree[i].val
    return tree


def with_field(tree, path, **kw):
    t = copy.deepcopy(tree)
    f = _parent(t, path[:-1])[path[-1]]
    for k, v in kw.items():
        setattr(f, k, v)
    return t


def inserted(tree, cpath, idx, field):
    t = copy.deepcopy(tree)
    _parent(t, cpath).insert(idx, field)
    return t


def removed(tree, path):
    t = copy.deepcopy(tree)
    del _parent(t, path[:-1])[path[-1]]
    return t


# ---- seeds (extreme values: 0, 127, 128, 2**63, 2**64 - 1) ----
def t_join(lt, id_):
    return [F(0x12, [F(0x09, lt), F(0x11, id_)])]


def t_leave(lt, id_, prune):
    return [F(0x0A, [F(0x09, lt)] + ([F(0x10, 1)] if prune else []) + [F(0x19, id_)])]


def t_user_event(name, pay):
    return ([F(0x0A, name)] if name else []) + ([F(0x12, pay)] if pay else [])


def t_push_pull(lt, status, left, ev, ring, q):
    body = [F(0x09, lt)] + [F(0x12, [F(0x09, k), F(0x11, v)]) for k, v in status] + [F(0x19, x) for x in left] + [F(0x21, ev)]
    body += [F(0x2A, [F(0x09, L)] + [F(0x12, t_user_event(n, p)) for n, p in evs]) for L, evs in ring]
    return [F(0x1A, body + [F(0x31, q)])]


def t_uem(lt, name, pay, cc):
    return [F(0x22, [F(0x09, lt)] + ([F(0x10, 1)] if cc else []) + ([F(0x1A, name)] if name else []) + ([F(0x22, pay)] if pay else []))]


M = 2**64 - 1
SEEDS = {
    "join": (t_join, (M, 128)),
    "leave_prune": (t_leave, (127, 2**63, True)),
    "leave": (t_leave, (0, M, False)),
    "push_pull": (t_push_pull, (128, [(0, M), (2**63, 127)], [2**63], 0, [], M)),
    "push_pull_ring": (t_push_pull, (2**63, [(127, 128)], [], M, [(128, [(b"deploy", b"v2"), (b"", b"\x00\xff")]), (M, [(b"x", b"")])], 0)),
    "uem_cc": (t_uem, (M, b"name", b"\x80\x00", True)),
    "uem": (t_uem, (128, b"n", b"", False)),
}


def seed_tree(name):
    fn, args = SEEDS[name]
    return fn(*args)


# ---- rewrites ----
def varint_forms(v):
    """(label, bytes) replacements of a varint: a canonical value of every length 1-10 (the smallest and the largest), the 10th
    byte 01 (accepted) and 02 / 7F / 81 (rejected), 11 bytes, and overlong zero-padded encodings (accepted)."""
    out = []
    for L in range(1, 11):
        lo, hi = (0 if L == 1 else 1 << 7 * (L - 1)), min((1 << 7 * L) - 1, M)
        out += [(("len", L, "min"), R.varint(lo)), (("len", L, "max"), R.varint(hi))]
    out += [(("tenth", x), b"\xff" * 9 + bytes([x])) for x in (0x01, 0x02, 0x7F, 0x81)]
    out += [(("eleven", "ff"), b"\xff" * 10 + b"\x01"), (("eleven", "80"), b"\x80" * 10 + b"\x00")]
    out += [(("overlong", "80 00"), b"\x80\x00"), (("overlong", "ff 80 00"), b"\xff\x80\x00"), (("overlong", "80x9 00"), b"\x80" * 9 + b"\x00")]
    c = R.varint(v)
    for k in (1, 2):
        if len(c) + k <= 10:
            out.append((("overlong", "pad", k), c[:-1] + bytes([c[-1] | 0x80]) + b"\x80" * (k - 1) + b"\x00"))
    return out


LEN_FORMS = {                                    # declared length of a length-delimited field: f(value bytes n, bytes left rem)
    "rem": lambda n, rem: R.varint(rem),
    "rem+1": lambda n, rem: R.varint(rem + 1),
    "n-1": lambda n, rem: R.varint(max(n - 1, 0)),
    "2^32-1": lambda n, rem: R.varint(2**32 - 1),
    "2^32": lambda n, rem: R.varint(2**32),
    "2^64-1": lambda n, rem: R.varint(M),
    "overlong": lambda n, rem: (lambda c: c[:-1] + bytes([c[-1] | 0x80, 0]))(R.varint(n)),
}
UNKNOWN_TAG = 15 << 3                            # a tag number no message of the path uses
UNKNOWN = {0: b"\x05", 1: b"\xac\x02", 2: b"\x03\x01\x02\x03", 3: b"\x01\x02\x03\x04", 4: bytes(range(8)), 5: b"\x00", 6: b"\x00", 7: b"\x00"}
UNKNOWN_CUT = {0: b"", 1: b"\x80", 2: b"\x03\x01", 3: b"\x01\x02", 4: bytes(range(7))}     # the same, cut short: only as a last field


class Case:
    __slots__ = ("seed", "family", "attr", "data")

    def __init__(self, seed, family, attr, data):
        self.seed, self.family, self.attr, self.data = seed, family, attr, data

    def __repr__(self):
        return f"Case({self.seed}, {self.family}, {self.attr}, {self.data.hex()})"


def corpus():
    cases = []
    for sname in SEEDS:
        tree = seed_tree(sname)
        b = ser(tree)
        cases.append(Case(sname, "seed", (), b))
        cases += [Case(sname, "truncate", (k,), b[:k]) for k in range(len(b))]
        for path, f in walk(tree):
            w = f.tag & 7
            if f.raw is None and w == VARINT:
                cases += [Case(sname, "varint", (path,) + lab, ser(with_field(tree, path, raw=raw))) for lab, raw in varint_forms(f.val)]
            if w == BYTE:
                cases += [Case(sname, "byte", (path, x), ser(with_field(tree, path, val=x))) for x in (0, 2, 0x80, 0xFF)]
            if w == LEN:
                cases += [Case(sname, "len", (path, lab), ser(with_field(tree, path, prefix=fn))) for lab, fn in LEN_FORMS.items()]
            cases += [Case(sname, "retype", (path, w2), ser(with_field(tree, path, tag=(f.tag & ~7) | w2, raw=enc(f, 0)[1:]))) for w2 in range(8) if w2 != w]
            cases.append(Case(sname, "duplicate", (path,), ser(inserted(tree, path[:-1], path[-1] + 1, copy.deepcopy(f)))))
            # a second copy cut short, as the last field: a duplicate of a singular field is reported before its value is read
            cut = {BYTE: b"", VARINT: b"\x80", LEN: b"\x05"}.get(w, b"")
            cases.append(Case(sname, "duplicate_cut", (path,), ser(inserted(tree, path[:-1], len(_parent(tree, path[:-1])), F(f.tag, raw=cut)))))
            cases.append(Case(sname, "remove", (path,), ser(removed(tree, path))))
        for cpath, cont in containers(tree):
            for idx in range(len(cont) + 1):
                cases += [Case(sname, "unknown", (cpath, idx, w), ser(inserted(tree, cpath, idx, F(UNKNOWN_TAG | w, raw=UNKNOWN[w])))) for w in range(8)]
            cases += [Case(sname, "unknown_cut", (cpath, w), ser(inserted(tree, cpath, len(cont), F(UNKNOWN_TAG | w, raw=UNKNOWN_CUT[w])))) for w in range(5)]
    for a in SEEDS:                              # two messages in one envelope, every pair of seeds in both orders
        for b in SEEDS:
            first, second = ser(seed_tree(a)), ser(seed_tree(b))
            cases.append(Case(a, "two", (b,), first + second))
            cases += [Case(a, "two_cut", (b, k), first + second[:k]) for k in range(1, len(second))]
    return cases


def capacity_message(n_status, n_left, ring_sizes):
    """A PushPull with n_status status entries, n_left left entries and one ring entry of ring_sizes[k] events per k."""
    status = [(i * 977 + 1, i) for i in range(n_status)]
    ring = [(k + 1, [(b"e%d" % j, b"") for j in range(m)]) for k, m in enumerate(ring_sizes)]
    return R.push_pull(5, status, list(range(100, 100 + n_left)), 6, ring, 7), status, ring


# ---- the three decoders, as outcomes: ("ok", value) or ("err", class) ----
PRODUCT_CLASSES = {b"truncated message": "truncated", b"varint longer than 64 bits": "varint", b"duplicate field": "duplicate",
                   b"missing field": "missing", b"unknown wire type": "wire_type", b"output capacity too small": "capacity",
                   b"not a message of the requested type": "type"}
ORACLE_CLASSES = {-1: "malformed", -3: "duplicate", -4: "missing", -6: "capacity", -7: "type"}
RESTATED_CLASSES = {"truncated": "truncated", "varint": "varint", "duplicate": "duplicate", "missing": "missing", "wire type": "wire_type", "type": "type"}
COARSE = {"truncated": "malformed", "varint": "malformed", "wire_type": "malformed"}


def product_class(text):
    for k, v in PRODUCT_CLASSES.items():
        if text.endswith(b"wire: " + k):
            return v
    raise AssertionError(f"unclassified product error: {text!r}")


def _p(P, rc, value):
    return ("ok", value) if rc == 0 else ("err", product_class(P.serfsim_last_error()))


def p_decode_push_pull(P, b, cap=BIG, left_cap=BIG):
    """serfsim_wire_decode_push_pull with separate status / left capacities."""
    ids, sts, left = np.zeros(max(cap, 1), np.uint64), np.zeros(max(cap, 1), np.uint64), np.zeros(max(left_cap, 1), np.uint64)
    m = W.PushPull(0, 0, 0, cap, left_cap, 0, 0, ids.ctypes.data_as(W.u64p), sts.ctypes.data_as(W.u64p), left.ctypes.data_as(W.u64p))
    rc = P.serfsim_wire_decode_push_pull(W._buf(b), len(b), C.byref(m))
    if rc:
        return rc, None
    return 0, (m.ltime, [(int(ids[i]), int(sts[i])) for i in range(m.n_status)], [int(x) for x in left[:m.n_left]], m.event_ltime, m.query_ltime, m.n_events_skipped)


def product(P, b):
    t = C.c_uint32()
    out = {"type": _p(P, P.serfsim_wire_message_type(W._buf(b), len(b), C.byref(t)), t.value)}
    out["intent"] = _p(P, *W.p_decode_intent(P, b))
    out["push_pull"] = _p(P, *p_decode_push_pull(P, b))
    out["ring"] = _p(P, *WE.decode_push_pull(P, b, cap=BIG, ring_cap=BIG, ev_cap=BIG))
    out["uem"] = _p(P, *WE.decode_user_event(P, b))
    return out


def oracle(b):
    rc, v = W.o_decode_intent(b)
    out = {"intent": ("ok", v) if rc == 0 else ("err", ORACLE_CLASSES[rc])}
    rc, v = W.o_decode_push_pull(b, cap=BIG)
    out["push_pull"] = ("ok", v) if rc == 0 else ("err", ORACLE_CLASSES[rc])
    return out


def _r(fn, b):
    try:
        return "ok", fn(b)
    except R.WireError as e:
        return "err", RESTATED_CLASSES[str(e)]


def restated(b):
    return {"type": _r(lambda x: R.open_envelope(x)[0], b), "intent": _r(R.d_intent, b), "ring": _r(R.d_push_pull, b), "uem": _r(R.d_user_event_message, b)}


def top_level_tags(b):
    """The tag bytes of the envelope stream up to its first framing error."""
    tags, o = [], 0
    try:
        while o < len(b):
            t = b[o]
            tags.append(t)
            w = t & 7
            if w == BYTE:
                o += 2
            elif w == VARINT:
                _, o = R.get_varint(b, o + 1)
            elif w == LEN:
                n, o = R.get_varint(b, o + 1)
                o += n
            elif w in (3, 4):
                o += 5 if w == 3 else 9
            else:
                break
    except R.WireError:
        pass
    return tags


def coarse(outcome):
    kind, v = outcome
    return (kind, COARSE.get(v, v)) if kind == "err" else outcome


def disagreements(P, b):
    """Every disagreement between the decoders on b that the documented differences do not explain."""
    p, o, r = product(P, b), oracle(b), restated(b)
    bad = []
    for k in ("type", "intent", "uem"):
        if p[k] != r[k]:
            bad.append((k, "product", p[k], "restatement", r[k]))
    ring = r["ring"]
    if ring[0] == "ok":
        lt, status, left, ev, rg, q = ring[1]
        ring = ("ok", (lt, status, left, ev, [(L, [(bytes(n), bytes(pl)) for n, pl in evs]) for L, evs in rg], q))
    if p["ring"] != ring:
        bad.append(("ring", "product", p["ring"], "restatement", ring))
    if 0x22 not in top_level_tags(b):            # the oracle does not know the UserEventMessage byte
        for k in ("intent", "push_pull"):
            if coarse(p[k]) != o[k]:
                bad.append((k, "product", p[k], "oracle", o[k]))
    return bad


# ---- what the batch kernels must give, from the host decoders ----
def expect_decode_batch(P, b, cap):
    """serfsim_wire_decode_batch on message b: ("ok", (ltime, status entries)) or ("err", class)."""
    rc, v = p_decode_push_pull(P, b, cap=cap, left_cap=MAX_SLOTS)
    return ("ok", (v[0], v[1])) if rc == 0 else ("err", product_class(P.serfsim_last_error()))


def ring_to_seen(ring, table):
    """(seen mask, unmatched count) of a decoded ring: tracked event e matches a UserEvent with its name and payload in an
    entry whose ltime is e's (non-zero) Lamport time; equal content and ltime → the lowest e."""
    names, pays, lts = table
    mask = um = 0
    for L, evs in ring:
        for n, p in evs:
            e = next((e for e in range(len(names)) if lts[e] and lts[e] == L and names[e] == n and pays[e] == p), None)
            if e is None:
                um += 1
            else:
                mask |= 1 << e
    return mask, um


def expect_events_batch(P, b, table):
    """serfsim_wire_decode_events_batch on message b: ("ok", (event_ltime, seen, unmatched)) or ("err", class)."""
    rc, v = WE.decode_push_pull(P, b, cap=BIG, ring_cap=BIG, ev_cap=BIG)
    if rc:
        return "err", product_class(P.serfsim_last_error())
    return ("ok", (v[3],) + ring_to_seen(v[4], table))


def pack(msgs):
    off = np.zeros(len(msgs) + 1, np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs], dtype=np.uint64)
    buf = np.frombuffer(b"".join(msgs), np.uint8) if msgs and off[-1] else np.zeros(0, np.uint8)
    return buf, off


_BATCH_ERR = re.compile(rb"wire: message (\d+): (.*)$")


def batch_error(text):
    """(first bad index, class) from the error text of a failed batch call."""
    m = _BATCH_ERR.search(text if isinstance(text, bytes) else text.encode())
    assert m, text
    return int(m.group(1)), product_class(m.group(2))


def run_decode_batch(P, sim, msgs, cap):
    """("ok", [(ltime, status)] per message) or ("err", index, class)."""
    buf, off = pack(msgs)
    rc, (lt, ids, sts, ns) = W.decode_batch(P, sim, buf, off, cap, check=False)
    if rc:
        return ("err",) + batch_error(P.serfsim_last_error())
    return "ok", [(int(lt[i]), [(int(ids[i, j]), int(sts[i, j])) for j in range(ns[i])]) for i in range(len(msgs))]


def run_events_batch(sim, msgs):
    """("ok", [(event_ltime, seen, unmatched)] per message) or ("err", index, class)."""
    from serf_b200.sim import SerfsimError
    buf, off = pack(msgs)
    try:
        ev, seen, um = sim.wire_decode_events(buf, off)
    except SerfsimError as e:
        return ("err",) + batch_error(str(e))
    return "ok", [(int(ev[i]), int(seen[i]), int(um[i])) for i in range(len(msgs))]


def check_in_batches(P, sim, table, cap, b, valid, k):
    """Message b alone and at index k of `valid` through both batch kernels: the call fails at the first bad index with the
    host decoder's class, or decodes every message as the host decoders do."""
    for msgs, at in (([b], 0), (valid[:k] + [b] + valid[k:], k)):
        want = [expect_decode_batch(P, m, cap) for m in msgs]
        got = run_decode_batch(P, sim, msgs, cap)
        bad = [i for i, w in enumerate(want) if w[0] == "err"]
        if bad:
            assert bad == [at] and got == ("err", at, want[at][1]), (b.hex(), at, got, want[at])
        else:
            assert got == ("ok", [w[1] for w in want]), (b.hex(), at, got)
        want = [expect_events_batch(P, m, table) for m in msgs]
        got = run_events_batch(sim, msgs)
        bad = [i for i, w in enumerate(want) if w[0] == "err"]
        if bad:
            assert bad == [at] and got == ("err", at, want[at][1]), (b.hex(), at, got, want[at])
        else:
            assert got == ("ok", [w[1] for w in want]), (b.hex(), at, got)
