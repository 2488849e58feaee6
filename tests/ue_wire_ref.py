"""An independent restatement, in Python, of user events on serf's wire — test infrastructure, the checker of the user-event
half of serf_b200/csrc/wire.cuh / wire_codec.cu, and the third decoder (beside the product and oracle/wire_oracle.cpp) of
Join / Leave / PushPull that tests/test_wire_malformed.py compares on malformed bytes.

Follows serf-core/src/types: user_event.rs (UserEvent: name = 1, payload = 2, LengthDelimited, each written only when
non-empty, both default to empty, a second one is a duplicate), user_event/user_events.rs (UserEvents: ltime = 1 Varint
required, events = 2 repeated LengthDelimited UserEvent), user_event/message.rs (UserEventMessage: ltime = 1, cc = 2 Byte,
name = 3, payload = 4; encoded ltime, cc only when true, name, payload), message.rs:17-47 / 397-428 / 507-692 (message byte
merge(LengthDelimited, tag) + varint length; one message per buffer) and push_pull.rs:455-587 (PushPull `events` = 5: one
UserEvents per occupied ring slot, written between event_ltime and query_ltime).  The byte layout of memberlist_core::proto
(tag byte = tag << 3 | wire type, LEB128 varints, [varint length][bytes] for strings, bytes and nested messages) is restated
from the protobuf conventions that crate follows, as in oracle/wire_oracle.cpp: UNPINNED at byte level.

Expected per-node rings come from the oracle's state (the seen mask of its event records and the Lamport time of every tracked
event): one slot per distinct ltime % 512, slots ascending, events in a slot by ascending tracked index — the modelling rule of
DESIGN §8.4 (the reference keeps arrival order inside a slot; the packed record keeps none)."""
BYTE, VARINT, LEN = 0, 1, 2


def tag(wire, t):
    return t << 3 | wire


MSG = {1: "leave", 2: "join", 3: "push_pull", 4: "user_event"}
MSG_BYTES = {tag(LEN, t) for t in MSG}


class WireError(Exception):
    pass


def varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def get_varint(b, o):
    v = 0
    for i in range(10):
        if o + i >= len(b):
            raise WireError("truncated")
        c = b[o + i]
        if i == 9 and c > 1:
            raise WireError("varint")
        v |= (c & 0x7F) << (7 * i)
        if not c & 0x80:
            return v, o + i + 1
    raise WireError("varint")


def fields(b, once=None):
    """(tag byte, value) for every field of a TLV stream: int for Varint / Byte, bytes for LengthDelimited.  once: tag byte →
    group of the fields that may appear once; a second field of a group is a duplicate, reported before its value is read
    (the `if x.is_some() { return Err(duplicate_field) }` that opens every singular arm, e.g. join.rs:68-75, message.rs:520-527)."""
    o, seen = 0, set()
    while o < len(b):
        t = b[o]
        w = t & 7
        if once and t in once:
            if once[t] in seen:
                raise WireError("duplicate")
            seen.add(once[t])
        o += 1
        if w == BYTE:
            if o >= len(b):
                raise WireError("truncated")
            yield t, b[o]
            o += 1
        elif w == VARINT:
            v, o = get_varint(b, o)
            yield t, v
        elif w == LEN:
            n, o = get_varint(b, o)
            if len(b) - o < n:
                raise WireError("truncated")
            yield t, bytes(b[o:o + n])
            o += n
        elif w == 3 or w == 4:
            n = 4 if w == 3 else 8
            if len(b) - o < n:
                raise WireError("truncated")
            yield t, bytes(b[o:o + n])
            o += n
        else:
            raise WireError("wire type")


def ld(t, v):
    return bytes([t]) + varint(len(v)) + bytes(v)


def envelope(msg_tag, body):
    return ld(tag(LEN, msg_tag), body)


# ---- encoders ----
def user_event(name, payload):
    return (ld(tag(LEN, 1), name) if name else b"") + (ld(tag(LEN, 2), payload) if payload else b"")


def user_events(ltime, events):
    return bytes([tag(VARINT, 1)]) + varint(ltime) + b"".join(ld(tag(LEN, 2), user_event(n, p)) for n, p in events)


def user_event_message(ltime, name, payload, cc):
    body = bytes([tag(VARINT, 1)]) + varint(ltime) + (bytes([tag(BYTE, 2), 1]) if cc else b"")
    body += (ld(tag(LEN, 3), name) if name else b"") + (ld(tag(LEN, 4), payload) if payload else b"")
    return envelope(4, body)


def push_pull(ltime, status, left, event_ltime, ring, query_ltime):
    """ring: [(ltime, [(name, payload), ...]), ...] in the order the message carries it."""
    body = bytes([tag(VARINT, 1)]) + varint(ltime)
    for k, v in status:
        body += ld(tag(LEN, 2), bytes([tag(VARINT, 1)]) + varint(k) + bytes([tag(VARINT, 2)]) + varint(v))
    for k in left:
        body += bytes([tag(VARINT, 3)]) + varint(k)
    body += bytes([tag(VARINT, 4)]) + varint(event_ltime)
    for lt, evs in ring:
        body += ld(tag(LEN, 5), user_events(lt, evs))
    body += bytes([tag(VARINT, 6)]) + varint(query_ltime)
    return envelope(3, body)


# ---- decoders (raise WireError) ----
def _once(*tags):
    return {t: t for t in tags}


def open_envelope(b):
    found = None
    for t, v in fields(b, once={t: "message" for t in MSG_BYTES}):          # one message per buffer (message.rs:520-527)
        if t in MSG_BYTES:
            found = (t >> 3, v)
    if found is None:
        raise WireError("missing")
    return found


def d_intent(b):
    """JoinMessage::decode (join.rs:54-105) / LeaveMessage::decode (leave.rs:56-119) with the envelope: (kind, ltime, id,
    prune), kind 1 = leave, 2 = join.  A second Join id is a duplicate; a second Leave id replaces the first."""
    kind, body = open_envelope(b)
    if kind not in (1, 2):
        raise WireError("type")
    leave = kind == 1
    if leave:                                                  # leave.rs:8-13: ltime = 1, prune = 2 (Byte), id = 3
        keys, once = {tag(VARINT, 1): "ltime", tag(BYTE, 2): "prune", tag(VARINT, 3): "id"}, _once(tag(VARINT, 1), tag(BYTE, 2))
    else:                                                      # join.rs:8-10: ltime = 1, id = 2
        keys, once = {tag(VARINT, 1): "ltime", tag(VARINT, 2): "id"}, _once(tag(VARINT, 1), tag(VARINT, 2))
    got = {}
    for t, v in fields(body, once=once):
        if t in keys:
            got[keys[t]] = v
    if "ltime" not in got or "id" not in got:
        raise WireError("missing")
    return kind, got["ltime"], got["id"], bool(got.get("prune", 0))


def d_user_event(b):
    name = payload = None
    for t, v in fields(b, once=_once(tag(LEN, 1), tag(LEN, 2))):
        if t == tag(LEN, 1):
            name = v
        elif t == tag(LEN, 2):
            payload = v
    return name or b"", payload or b""


def d_user_events(b):
    lt, evs = None, []
    for t, v in fields(b, once=_once(tag(VARINT, 1))):
        if t == tag(VARINT, 1):
            lt = v
        elif t == tag(LEN, 2):
            evs.append(d_user_event(v))
    if lt is None:
        raise WireError("missing")
    return lt, evs


def d_user_event_message(b):
    kind, body = open_envelope(b)
    if kind != 4:
        raise WireError("type")
    keys = {tag(VARINT, 1): "ltime", tag(BYTE, 2): "cc", tag(LEN, 3): "name", tag(LEN, 4): "payload"}
    got = {}
    for t, v in fields(body, once=_once(*keys)):
        if t in keys:
            got[keys[t]] = v
    if "ltime" not in got:
        raise WireError("missing")
    return got["ltime"], got.get("name", b""), got.get("payload", b""), bool(got.get("cc", 0))


def d_push_pull(b):
    kind, body = open_envelope(b)
    if kind != 3:
        raise WireError("type")
    one, status, left, ring = {}, [], [], []
    for t, v in fields(body, once=_once(tag(VARINT, 1), tag(VARINT, 4), tag(VARINT, 6))):
        if t in (tag(VARINT, 1), tag(VARINT, 4), tag(VARINT, 6)):
            one[t] = v
        elif t == tag(LEN, 2):
            kv = dict((tt, vv) for tt, vv in fields(v) if tt in (tag(VARINT, 1), tag(VARINT, 2)))
            if len(kv) != 2:
                raise WireError("missing")
            status.append((kv[tag(VARINT, 1)], kv[tag(VARINT, 2)]))
        elif t == tag(VARINT, 3):
            left.append(v)
        elif t == tag(LEN, 5):
            ring.append(d_user_events(v))
    if len(one) != 3:
        raise WireError("missing")
    return one[tag(VARINT, 1)], status, left, one[tag(VARINT, 4)], ring, one[tag(VARINT, 6)]


# ---- the simulator's rings ----
def ring_of(seen_mask, ltimes, contents):
    """The ring a node with tracked events `seen_mask` holds: [(slot ltime, [(name, payload), ...])] by ascending ring index,
    events of a slot by ascending tracked index.  ltimes[e]: Lamport time of tracked event e; contents[e]: (name, payload)."""
    slots = {}
    for e in range(len(ltimes)):
        if (seen_mask >> e) & 1:
            slots.setdefault(int(ltimes[e]) % 512, []).append(e)
    return [(int(ltimes[es[0]]), [contents[e] for e in es]) for _, es in sorted(slots.items())]
