"""ctypes glue shared by the wire-codec tests: the oracle's restatement (oracle/wire_oracle.cpp) and the product's C ABI."""
import ctypes as C

import numpy as np

from oracle_lib import lib as oracle_lib

u8p, u64p, u32p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)
LEAVE, JOIN, PUSH_PULL = 1, 2, 3


class Intent(C.Structure):                       # serfsim_wire_intent_t
    _fields_ = [("type", C.c_uint32), ("prune", C.c_uint32), ("ltime", C.c_uint64), ("id", C.c_uint64)]


class PushPull(C.Structure):                     # serfsim_wire_push_pull_t
    _fields_ = [("ltime", C.c_uint64), ("event_ltime", C.c_uint64), ("query_ltime", C.c_uint64), ("n_status", C.c_uint32), ("n_left", C.c_uint32),
                ("n_events_skipped", C.c_uint32), ("pad", C.c_uint32), ("status_ids", u64p), ("status_ltimes", u64p), ("left_ids", u64p)]


def _oracle():
    L = oracle_lib()
    L.oracle_wire_encode_intent.restype, L.oracle_wire_encode_intent.argtypes = C.c_int, [C.c_uint32, C.c_uint64, C.c_uint64, C.c_int, u8p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.oracle_wire_decode_intent.restype, L.oracle_wire_decode_intent.argtypes = C.c_int, [u8p, C.c_size_t, u32p, u64p, u64p, C.POINTER(C.c_int)]
    L.oracle_wire_encode_push_pull.restype = C.c_int
    L.oracle_wire_encode_push_pull.argtypes = [C.c_uint64, u64p, u64p, C.c_uint32, u64p, C.c_uint32, C.c_uint64, C.c_uint64, u8p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.oracle_wire_decode_push_pull.restype = C.c_int
    L.oracle_wire_decode_push_pull.argtypes = [u8p, C.c_size_t, u64p, u64p, u64p, u32p, u64p, u32p, u64p, u64p, u32p]
    return L


def _buf(b):
    return (C.c_uint8 * max(1, len(b))).from_buffer_copy(bytes(b) or b"\0")


def _arr(v):
    a = np.ascontiguousarray(v, dtype=np.uint64)
    return a, a.ctypes.data_as(u64p)


# ---- oracle ----
def o_encode_intent(type_, ltime, id_, prune=False):
    L = _oracle()
    out, n = (C.c_uint8 * 64)(), C.c_size_t()
    assert L.oracle_wire_encode_intent(type_, ltime, id_, int(prune), out, 64, C.byref(n)) == 0
    return bytes(out[:n.value])


def o_decode_intent(b):
    L = _oracle()
    t, lt, id_, pr = C.c_uint32(), C.c_uint64(), C.c_uint64(), C.c_int()
    rc = L.oracle_wire_decode_intent(_buf(b), len(b), C.byref(t), C.byref(lt), C.byref(id_), C.byref(pr))
    return rc, (t.value, lt.value, id_.value, bool(pr.value))


def o_encode_push_pull(ltime, status, left, event_ltime, query_ltime):
    L = _oracle()
    ids, pi = _arr([k for k, _ in status]); sts, ps = _arr([v for _, v in status]); lf, pl = _arr(left)
    cap = 64 + 24 * (len(status) + len(left))
    out, n = (C.c_uint8 * cap)(), C.c_size_t()
    assert L.oracle_wire_encode_push_pull(ltime, pi, ps, len(status), pl, len(left), event_ltime, query_ltime, out, cap, C.byref(n)) == 0
    return bytes(out[:n.value])


def o_decode_push_pull(b, cap=64):
    L = _oracle()
    ids, sts, left = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    lt, ev, q = C.c_uint64(), C.c_uint64(), C.c_uint64()
    ns, nl, ne = C.c_uint32(cap), C.c_uint32(cap), C.c_uint32()
    rc = L.oracle_wire_decode_push_pull(_buf(b), len(b), C.byref(lt), ids.ctypes.data_as(u64p), sts.ctypes.data_as(u64p), C.byref(ns), left.ctypes.data_as(u64p), C.byref(nl),
                                        C.byref(ev), C.byref(q), C.byref(ne))
    if rc:
        return rc, None
    return 0, (lt.value, [(int(ids[i]), int(sts[i])) for i in range(ns.value)], [int(x) for x in left[:nl.value]], ev.value, q.value, ne.value)


# ---- product (any library exporting the serfsim_wire_* entry points: libserfsim.so, or its host build of tests/emu) ----
def bind_product(L):
    L.serfsim_wire_encoded_len_intent.restype, L.serfsim_wire_encoded_len_intent.argtypes = C.c_size_t, [C.POINTER(Intent)]
    L.serfsim_wire_encode_intent.restype, L.serfsim_wire_encode_intent.argtypes = C.c_int, [C.POINTER(Intent), u8p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.serfsim_wire_encode_push_pull.restype, L.serfsim_wire_encode_push_pull.argtypes = C.c_int, [C.POINTER(PushPull), u8p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.serfsim_wire_message_type.restype, L.serfsim_wire_message_type.argtypes = C.c_int, [u8p, C.c_size_t, u32p]
    L.serfsim_wire_decode_intent.restype, L.serfsim_wire_decode_intent.argtypes = C.c_int, [u8p, C.c_size_t, C.POINTER(Intent)]
    L.serfsim_wire_decode_push_pull.restype, L.serfsim_wire_decode_push_pull.argtypes = C.c_int, [u8p, C.c_size_t, C.POINTER(PushPull)]
    L.serfsim_wire_local_state_batch.restype = C.c_int
    L.serfsim_wire_local_state_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t)]
    L.serfsim_wire_decode_batch.restype = C.c_int
    L.serfsim_wire_decode_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def p_encode_intent(L, type_, ltime, id_, prune=False):
    m = Intent(type_, int(prune), ltime, id_)
    need = L.serfsim_wire_encoded_len_intent(C.byref(m))
    out, n = (C.c_uint8 * need)(), C.c_size_t()
    assert L.serfsim_wire_encode_intent(C.byref(m), out, need, C.byref(n)) == 0 and n.value == need
    return bytes(out)


def p_decode_intent(L, b):
    m = Intent()
    rc = L.serfsim_wire_decode_intent(_buf(b), len(b), C.byref(m))
    return rc, (m.type, m.ltime, m.id, bool(m.prune))


def p_encode_push_pull(L, ltime, status, left, event_ltime, query_ltime):
    ids, pi = _arr([k for k, _ in status]); sts, ps = _arr([v for _, v in status]); lf, pl = _arr(left)
    m = PushPull(ltime, event_ltime, query_ltime, len(status), len(left), 0, 0, pi, ps, pl)
    n = C.c_size_t()
    L.serfsim_wire_encode_push_pull(C.byref(m), None, 0, C.byref(n))             # sizing call: fails, reports the needed size
    out = (C.c_uint8 * n.value)()
    assert L.serfsim_wire_encode_push_pull(C.byref(m), out, n.value, C.byref(n)) == 0
    return bytes(out)


def p_decode_push_pull(L, b, cap=64):
    ids, sts, left = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    m = PushPull(0, 0, 0, cap, cap, 0, 0, ids.ctypes.data_as(u64p), sts.ctypes.data_as(u64p), left.ctypes.data_as(u64p))
    rc = L.serfsim_wire_decode_push_pull(_buf(b), len(b), C.byref(m))
    if rc:
        return rc, None
    return 0, (m.ltime, [(int(ids[i]), int(sts[i])) for i in range(m.n_status)], [int(x) for x in left[:m.n_left]], m.event_ltime, m.query_ltime, m.n_events_skipped)


def local_state_batch(L, sim):
    """All push-pull messages of the shard, encoded by the kernels; returns (bytes, offsets)."""
    n = sim.count
    off = np.zeros(n + 1, np.uint64)
    tot = C.c_size_t()
    L.serfsim_wire_local_state_batch(sim._h, None, 0, off.ctypes.data, C.byref(tot))       # sizing call
    out = np.zeros(max(1, tot.value), np.uint8)
    rc = L.serfsim_wire_local_state_batch(sim._h, out.ctypes.data, out.size, off.ctypes.data, C.byref(tot))
    assert rc == 0, rc
    return out[:tot.value], off


def decode_batch(L, sim, buf, off, cap, check=True):
    """serfsim_wire_decode_batch over message i = buf[off[i]:off[i + 1]].  check=False returns (rc, outputs) instead of
    asserting success."""
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    if off.ndim != 1 or off.size == 0:
        raise ValueError("offsets must be a 1-D array of n + 1 entries")
    if int(off[-1]) > buf.size:
        raise ValueError(f"offsets[-1] = {int(off[-1])} is past the end of the {buf.size}-byte buffer")
    n = off.size - 1
    lt, ids, sts, ns = np.zeros(n, np.uint64), np.zeros((n, cap), np.uint64), np.zeros((n, cap), np.uint64), np.zeros(n, np.uint32)
    rc = L.serfsim_wire_decode_batch(sim._h, buf.ctypes.data, off.ctypes.data, n, cap, lt.ctypes.data, ids.ctypes.data, sts.ctypes.data, ns.ctypes.data)
    if not check:
        return rc, (lt, ids, sts, ns)
    assert rc == 0, rc
    return lt, ids, sts, ns


def expected_local_state(sim_like, v_local, subjects):
    """What SerfDelegate::local_state of local node v holds, from the driver's getters (oracle or device)."""
    status, ltimes = [], []
    left = []
    for s, subj in enumerate(subjects):
        st = sim_like["status"][s][v_local]
        if st != 0:                                            # MemberStatus::None = not in the member table
            status.append((int(subj), int(sim_like["ltime"][s][v_local])))
            if st == 3:
                left.append(int(subj))
    return int(sim_like["clock"][v_local]), status, left
