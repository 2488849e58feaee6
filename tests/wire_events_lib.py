"""ctypes glue for the user-event half of the product's wire codec (include/serfsim.h): UserEventMessage and PushPull with
the event ring, on any library exporting the serfsim_wire_* entry points (libserfsim.so, or its host build of tests/emu)."""
import ctypes as C

import numpy as np

import wire_lib as W

u8p = C.POINTER(C.c_uint8)
USER_EVENT = 4


class UserEventMsg(C.Structure):                 # serfsim_wire_user_event_t
    _fields_ = [("ltime", C.c_uint64), ("name", u8p), ("name_len", C.c_size_t), ("payload", u8p), ("payload_len", C.c_size_t),
                ("cc", C.c_uint32), ("pad", C.c_uint32)]


class Event(C.Structure):                        # serfsim_wire_event_t
    _fields_ = [("name", u8p), ("name_len", C.c_size_t), ("payload", u8p), ("payload_len", C.c_size_t)]


class Slot(C.Structure):                         # serfsim_wire_user_events_t
    _fields_ = [("ltime", C.c_uint64), ("n_events", C.c_uint32), ("pad", C.c_uint32), ("events", C.POINTER(Event))]


def bind(L):
    W.bind_product(L)
    L.serfsim_wire_encode_user_event.restype = C.c_int
    L.serfsim_wire_encode_user_event.argtypes = [C.POINTER(UserEventMsg), u8p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.serfsim_wire_decode_user_event.restype = C.c_int
    L.serfsim_wire_decode_user_event.argtypes = [u8p, C.c_size_t, C.POINTER(UserEventMsg)]
    L.serfsim_wire_encode_push_pull_events.restype = C.c_int
    L.serfsim_wire_encode_push_pull_events.argtypes = [C.POINTER(W.PushPull), C.POINTER(Slot), C.c_uint32, u8p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.serfsim_wire_decode_push_pull_events.restype = C.c_int
    L.serfsim_wire_decode_push_pull_events.argtypes = [u8p, C.c_size_t, C.POINTER(W.PushPull), C.POINTER(Slot), C.POINTER(C.c_uint32),
                                                       C.POINTER(Event), C.POINTER(C.c_uint32)]
    return L


def _ptr(b, keep):
    if not b:
        return None
    buf = (C.c_uint8 * len(b)).from_buffer_copy(bytes(b))
    keep.append(buf)
    return C.cast(buf, u8p)


def _bytes(p, n):
    return C.string_at(p, n) if n else b""


def encode_user_event(L, ltime, name, payload, cc=False):
    keep = []
    m = UserEventMsg(ltime, _ptr(name, keep), len(name), _ptr(payload, keep), len(payload), int(cc), 0)
    n = C.c_size_t()
    rc = L.serfsim_wire_encode_user_event(C.byref(m), None, 0, C.byref(n))          # sizing call: fails, reports the size
    assert rc != 0
    out = (C.c_uint8 * max(1, n.value))()
    assert L.serfsim_wire_encode_user_event(C.byref(m), out, n.value, C.byref(n)) == 0
    return bytes(out[:n.value])


def decode_user_event(L, b):
    m = UserEventMsg()
    buf = W._buf(b)
    rc = L.serfsim_wire_decode_user_event(buf, len(b), C.byref(m))
    if rc:
        return rc, None
    return 0, (m.ltime, _bytes(m.name, m.name_len), _bytes(m.payload, m.payload_len), bool(m.cc))


def encode_push_pull(L, ltime, status, left, event_ltime, ring, query_ltime):
    keep = []
    ids, pi = W._arr([k for k, _ in status]); sts, ps = W._arr([v for _, v in status]); lf, pl = W._arr(left)
    m = W.PushPull(ltime, event_ltime, query_ltime, len(status), len(left), 0, 0, pi, ps, pl)
    slots = (Slot * max(1, len(ring)))()
    for k, (lt, evs) in enumerate(ring):
        arr = (Event * max(1, len(evs)))(*[Event(_ptr(nm, keep), len(nm), _ptr(py, keep), len(py)) for nm, py in evs])
        keep.append(arr)
        slots[k] = Slot(lt, len(evs), 0, arr if evs else None)
    n = C.c_size_t()
    L.serfsim_wire_encode_push_pull_events(C.byref(m), slots, len(ring), None, 0, C.byref(n))
    out = (C.c_uint8 * n.value)()
    assert L.serfsim_wire_encode_push_pull_events(C.byref(m), slots, len(ring), out, n.value, C.byref(n)) == 0
    return bytes(out)


def decode_push_pull(L, b, cap=64, ring_cap=64, ev_cap=256):
    ids, sts, left = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    m = W.PushPull(0, 0, 0, cap, cap, 7, 0, ids.ctypes.data_as(W.u64p), sts.ctypes.data_as(W.u64p), left.ctypes.data_as(W.u64p))
    slots, evs = (Slot * max(1, ring_cap))(), (Event * max(1, ev_cap))()
    nr, ne = C.c_uint32(ring_cap), C.c_uint32(ev_cap)
    buf = W._buf(b)
    rc = L.serfsim_wire_decode_push_pull_events(buf, len(b), C.byref(m), slots, C.byref(nr), evs, C.byref(ne))
    if rc:
        return rc, None
    assert m.n_events_skipped == 0
    ring = [(slots[k].ltime, [(_bytes(slots[k].events[j].name, slots[k].events[j].name_len),
                               _bytes(slots[k].events[j].payload, slots[k].events[j].payload_len)) for j in range(slots[k].n_events)])
            for k in range(nr.value)]
    assert sum(len(e) for _, e in ring) == ne.value
    return 0, (m.ltime, [(int(ids[i]), int(sts[i])) for i in range(m.n_status)], [int(x) for x in left[:m.n_left]], m.event_ltime, ring, m.query_ltime)
