"""ctypes mirror of include/serfsim.h.

`GossipSim` follows the reference's operator surface for the hot path:
  Serf::join / leave / remove_failed_node   (serf-core/src/serf/api.rs:318-361, 422-499, 505-515)
  Serf::members → MemberStatus per member   (serf/api.rs:136-146, types/member.rs:54-58)
  Serf::stats                               (serf/api.rs:150-183, 588-602)
with the SWIM fault injection the simulator adds (fail / rejoin).  All compute happens in
libserfsim.so on the GPU; if the library is missing or there is no CUDA device the calls
raise — there is no Python or CPU fallback.
"""
import ctypes as C
import enum
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ABI_VERSION = 4


class MemberStatus(enum.IntEnum):      # types/member.rs:54-58
    NONE = 0
    ALIVE = 1
    LEAVING = 2
    LEFT = 3
    FAILED = 4


class MlState(enum.IntEnum):           # memberlist node state (external crate)
    ALIVE = 0
    SUSPECT = 1
    DEAD = 2
    LEFT = 3


class Op(enum.IntEnum):                # SERFSIM_OP_*
    JOIN = 1
    LEAVE = 2
    FORCE_LEAVE = 3
    FAIL = 4
    REJOIN = 5
    USER_EVENT = 6                     # Serf::user_event, serf/api.rs:241-299
    FORCE_LEAVE_PRUNE = 7              # Serf::remove_failed_node_prune, serf/api.rs:513 (LeaveMessage.prune: receivers erase the member)


class Config(C.Structure):             # serfsim_config_t
    _fields_ = [("abi_version", C.c_uint32), ("n_nodes", C.c_uint32), ("slots", C.c_uint32), ("fanout", C.c_uint32),
                ("retransmit_mult", C.c_uint32), ("suspicion_mult", C.c_uint32), ("suspicion_max_timeout_mult", C.c_uint32),
                ("probe_interval_ticks", C.c_uint32), ("gossip_interval_ms", C.c_uint32), ("init_status_ltime", C.c_uint32),
                ("init_clock", C.c_uint32), ("trace", C.c_uint32), ("seed", C.c_uint64), ("device", C.c_int32),
                ("rank", C.c_int32), ("world_size", C.c_int32), ("push_pull_interval_ticks", C.c_int32),
                ("reap_interval_ticks", C.c_uint32), ("tombstone_timeout_ticks", C.c_uint32), ("reconnect_timeout_ticks", C.c_uint32),
                ("recent_intent_timeout_ticks", C.c_uint32)]


class Stats(C.Structure):              # serfsim_stats_t
    _fields_ = [(n, C.c_uint64) for n in ("tick", "packets", "edge_updates", "messages", "changed", "events", "pending",
                                          "last_active_tick", "members", "member_time", "intent_queue", "disagree_slots")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


class ByzantineStats(C.Structure):     # serfsim_byz_stats_t
    _fields_ = [(n, C.c_uint64) for n in ("messages", "edge_updates", "flagged")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class UserEventStats(C.Structure):     # serfsim_uevent_stats_t
    _fields_ = [(n, C.c_uint64) for n in ("messages", "edge_updates", "delivered", "duplicates", "too_old", "event_queue", "event_time")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


UEVENT_RECORD_DTYPE = np.dtype([("event_clock", "<u4"), ("seen", "u1"), ("first", "u1"), ("pad", "<u2"), ("tx", "u1", (8,))])
assert UEVENT_RECORD_DTYPE.itemsize == 16


class TickRow(C.Structure):            # serfsim_tick_row_t
    _fields_ = [(n, C.c_uint64) for n in ("packets", "edge_updates", "messages", "changed", "pending", "events", "suspects", "hash")]


TRACE_DTYPE = np.dtype([(n, "<u8") for n, _ in TickRow._fields_])
RECORD_DTYPE = np.dtype([("status_ltime", "<u4"), ("qjoin_lt", "<u4"), ("qleave_lt", "<u4"), ("incarnation", "<u4"),
                         ("deadline", "<u4"), ("leave_tick", "<u4"), ("status", "u1"), ("ml", "u1"), ("tx_join", "u1"),
                         ("tx_leave", "u1"), ("tx_ml", "u1"), ("flags", "u1"), ("conf_mask", "<u2")])
assert RECORD_DTYPE.itemsize == 32

EVENT_CB = C.CFUNCTYPE(None, C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32), C.c_uint32)
BARRIER_FN = C.CFUNCTYPE(None, C.c_void_p)
ALLREDUCE_FN = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(C.c_uint64), C.c_uint32)


class SerfsimError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"serfsim error {code}: {msg}")
        self.code = code


_vp, _u32, _u64 = C.c_void_p, C.c_uint32, C.c_uint64
# name → (restype, argtypes) for every entry point a handle-based driver needs (prefix-relative)
SIGNATURES = {
    "create": (C.c_int, [C.POINTER(Config), C.POINTER(_vp)]),
    "destroy": (None, [_vp]),
    "set_topology_csr": (C.c_int, [_vp, _vp, _vp]),
    "set_subjects": (C.c_int, [_vp, _vp]),
    "reset": (C.c_int, [_vp, _u64]),
    "inject": (C.c_int, [_vp, _u32, _u32, _u32, _u32]),
    "step": (C.c_int, [_vp, _u32]),
    "run_until_converged": (C.c_int, [_vp, _u32, C.POINTER(_u32)]),
    "member_status": (C.c_int, [_vp, _u32, _vp]),
    "status_ltime": (C.c_int, [_vp, _u32, _vp]),
    "lamport_time": (C.c_int, [_vp, _vp]),
    "status_ltime_u32": (C.c_int, [_vp, _u32, _vp]),
    "lamport_time_u32": (C.c_int, [_vp, _vp]),
    "incarnation": (C.c_int, [_vp, _u32, _vp]),
    "ml_state": (C.c_int, [_vp, _u32, _vp]),
    "records": (C.c_int, [_vp, _u32, _vp]),
    "stats": (C.c_int, [_vp, C.POINTER(Stats)]),
    "tick_trace": (C.c_int, [_vp, _u32, _u32, _vp]),
    "state_hash": (C.c_int, [_vp, C.POINTER(_u64)]),
    "set_byzantine": (C.c_int, [_vp, _u32, _vp, _u32]),
    "anomaly_flags": (C.c_int, [_vp, _vp]),
    "byzantine_stats": (C.c_int, [_vp, C.POINTER(ByzantineStats)]),
    "set_user_events": (C.c_int, [_vp, _u32, _vp]),
    "event_time": (C.c_int, [_vp, _vp]),
    "user_event_seen": (C.c_int, [_vp, _u32, _vp]),
    "user_event_ltime": (C.c_int, [_vp, _u32, C.POINTER(_u64)]),
    "user_event_records": (C.c_int, [_vp, _vp]),
    "user_event_stats": (C.c_int, [_vp, C.POINTER(UserEventStats)]),
}
PRODUCT_ONLY = {
    "serfsim_abi_version": (_u32, []),
    "serfsim_default_config": (None, [C.POINTER(Config)]),
    "serfsim_last_error": (C.c_char_p, []),
    "serfsim_shard_range": (C.c_int, [_vp, C.POINTER(_u32), C.POINTER(_u32)]),
    "serfsim_set_event_cb": (C.c_int, [_vp, EVENT_CB, _vp]),
    "serfsim_results_async": (C.c_int, [_vp, _u32, _vp, _vp, _vp]),
    "serfsim_results_wait": (C.c_int, [_vp]),
    "serfsim_last_step_device_ms": (C.c_int, [_vp, C.POINTER(C.c_double), C.POINTER(_u64)]),
    "serfsim_set_tick_timing": (C.c_int, [_vp, C.c_int]),
    "serfsim_tick_times": (C.c_int, [_vp, _u32, _u32, _vp]),
    "serfsim_tick_view_kinds": (C.c_int, [_vp, _u32, _u32, _vp]),
    "serfsim_comm_blob_size": (C.c_size_t, []),
    "serfsim_comm_export": (C.c_int, [_vp, _vp]),
    "serfsim_comm_connect": (C.c_int, [_vp, _vp]),
    "serfsim_comm_set_hooks": (C.c_int, [_vp, BARRIER_FN, ALLREDUCE_FN, _vp]),
    "serfsim_comm_loopback": (C.c_int, [_vp]),
    "serfsim_set_user_event_content": (C.c_int, [_vp, _u32, _vp, _vp, _vp, _vp]),
    "serfsim_wire_local_state_range": (C.c_int, [_vp, _u32, _u32, _vp, C.c_size_t, _vp, C.POINTER(C.c_size_t)]),
    "serfsim_wire_decode_events_batch": (C.c_int, [_vp, _vp, _vp, _u32, _vp, _vp, _vp]),
}

_LIB = None


def library_path():
    # SERFSIM_LIB: another nvcc build of the same sources (A/B measurements of kernel variants); same ABI check applies
    return os.environ.get("SERFSIM_LIB") or os.path.join(_HERE, "libserfsim.so")


def load_library():
    """Load libserfsim.so (the CUDA product).  Raises if it has not been built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if not os.path.exists(path):
        raise SerfsimError(-2, f"{path} is missing: build it with `python -m serf_b200.build` "
                               "(nvcc, sm_90a); there is no CPU fallback")
    lib = C.CDLL(path)
    if hasattr(lib, "emu_probe"):             # tests/emu's host-compiled build of the kernels is test infrastructure, never the product
        raise SerfsimError(-2, f"{path} is the host-compiled test build (tests/emu), not the CUDA library: refusing to use it as the product")
    for name, (res, args) in SIGNATURES.items():
        f = getattr(lib, "serfsim_" + name)
        f.restype, f.argtypes = res, args
    for name, (res, args) in PRODUCT_ONLY.items():
        f = getattr(lib, name)
        f.restype, f.argtypes = res, args
    if lib.serfsim_abi_version() != ABI_VERSION:
        raise SerfsimError(-1, "ABI version mismatch between sim.py and libserfsim.so")
    _LIB = lib
    return lib


def default_config(**kw):
    """memberlist LAN profile (serf-core/src/options.rs:521) in ticks; override by keyword."""
    cfg = Config(abi_version=ABI_VERSION, n_nodes=0, slots=1, fanout=3, retransmit_mult=4, suspicion_mult=4,
                 suspicion_max_timeout_mult=6, probe_interval_ticks=5, gossip_interval_ms=200, init_status_ltime=1,
                 init_clock=2, trace=0, seed=1, device=-1, rank=0, world_size=1, push_pull_interval_ticks=0,
                 reap_interval_ticks=0, tombstone_timeout_ticks=432000, reconnect_timeout_ticks=432000, recent_intent_timeout_ticks=1500)
    for k, v in kw.items():
        if not hasattr(cfg, k):
            raise TypeError(f"unknown config field {k}")
        setattr(cfg, k, v)
    return cfg


class GossipSim:
    """N virtual serf nodes × R tracked subjects on one GPU (or one shard of a multi-GPU run)."""

    def __init__(self, n_nodes, slots=1, _lib=None, _prefix="serfsim_", _errfn="serfsim_last_error", **cfg_kw):
        self._lib = _lib if _lib is not None else load_library()
        self._prefix = _prefix
        self._errfn = getattr(self._lib, _errfn)
        self.cfg = default_config(n_nodes=n_nodes, slots=slots, **cfg_kw)
        self.n = n_nodes
        self.slots = slots
        self._h = _vp()
        self._keep = []
        self._check(self._fn("create")(C.byref(self.cfg), C.byref(self._h)))
        self.first, self.count = 0, n_nodes
        if _prefix == "serfsim_":
            f, c = _u32(), _u32()
            self._check(self._lib.serfsim_shard_range(self._h, C.byref(f), C.byref(c)))
            self.first, self.count = f.value, c.value

    # -- plumbing ---------------------------------------------------------------------
    def _fn(self, name):
        return getattr(self._lib, self._prefix + name)

    def _check(self, rc):
        if rc < 0:
            msg = self._errfn()
            raise SerfsimError(rc, msg.decode() if msg else "")
        return rc

    def close(self):
        if self._h:
            self._fn("destroy")(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- setup ------------------------------------------------------------------------
    def set_topology(self, row_ptr, col_idx):
        row_ptr = np.ascontiguousarray(row_ptr, dtype=np.uint64)
        col_idx = np.ascontiguousarray(col_idx, dtype=np.uint32)
        assert row_ptr.shape == (self.n + 1,) and col_idx.shape == (int(row_ptr[-1]),)
        self._check(self._fn("set_topology_csr")(self._h, row_ptr.ctypes.data, col_idx.ctypes.data))

    def set_subjects(self, subjects):
        s = np.ascontiguousarray(subjects, dtype=np.uint32)
        assert s.shape == (self.slots,)
        self._check(self._fn("set_subjects")(self._h, s.ctypes.data))

    def reset(self, seed):
        self._check(self._fn("reset")(self._h, int(seed)))

    # -- host operations: the reference's API calls at their origin node ---------------
    def inject(self, tick, op, node, slot=0):
        self._check(self._fn("inject")(self._h, int(tick), int(op), int(node), int(slot)))

    def join(self, node, tick=0):               # Serf::join
        self.inject(tick, Op.JOIN, node)

    def leave(self, node, tick=0):              # Serf::leave
        self.inject(tick, Op.LEAVE, node)

    def remove_failed_node(self, origin, slot, tick=0):   # Serf::remove_failed_node (force_leave)
        self.inject(tick, Op.FORCE_LEAVE, origin, slot)

    def remove_failed_node_prune(self, origin, slot, tick=0):   # Serf::remove_failed_node_prune
        self.inject(tick, Op.FORCE_LEAVE_PRUNE, origin, slot)

    def fail(self, node, tick=0):
        self.inject(tick, Op.FAIL, node)

    def rejoin(self, node, tick=0):
        self.inject(tick, Op.REJOIN, node)

    # -- the hot path -----------------------------------------------------------------
    def step(self, n_ticks=1):
        self._check(self._fn("step")(self._h, int(n_ticks)))

    def run_until_converged(self, max_ticks=10000):
        t = _u32()
        rc = self._check(self._fn("run_until_converged")(self._h, int(max_ticks), C.byref(t)))
        return t.value, rc == 0

    # -- outputs ----------------------------------------------------------------------
    def _get(self, name, dtype, slot=None, out=None):
        if out is None:
            out = np.empty(self.count, dtype=dtype)
        assert out.dtype == np.dtype(dtype) and out.shape == (self.count,) and out.flags.c_contiguous
        if slot is None:
            self._check(self._fn(name)(self._h, out.ctypes.data))
        else:
            self._check(self._fn(name)(self._h, int(slot), out.ctypes.data))
        return out

    def member_status(self, slot=0, out=None): return self._get("member_status", np.uint8, slot, out)        # Serf::members
    def status_ltime(self, slot=0, out=None): return self._get("status_ltime", np.uint64, slot, out)
    def lamport_time(self, out=None): return self._get("lamport_time", np.uint64, None, out)
    def status_ltime_u32(self, slot=0, out=None): return self._get("status_ltime_u32", np.uint32, slot, out)       # same values, half the bytes
    def lamport_time_u32(self, out=None): return self._get("lamport_time_u32", np.uint32, None, out)
    def results_async(self, slot=0, status=None, status_ltime=None, lamport=None):
        """Queue the read-back of the step's result vectors into caller-owned (pinned) numpy arrays; returns the bytes queued."""
        ptr = lambda a: a.ctypes.data if a is not None else None
        self._check(self._lib.serfsim_results_async(self._h, int(slot), ptr(status), ptr(status_ltime), ptr(lamport)))
        return sum(a.nbytes for a in (status, status_ltime, lamport) if a is not None)

    def results_wait(self):
        self._check(self._lib.serfsim_results_wait(self._h))

    def incarnation(self, slot=0): return self._get("incarnation", np.uint32, slot)
    def ml_state(self, slot=0): return self._get("ml_state", np.uint8, slot)
    def records(self, slot=0): return self._get("records", RECORD_DTYPE, slot)

    # -- byzantine stale-record injectors (BASELINE configs[4]) ------------------------------
    def set_byzantine(self, ids, delta=2):
        a = np.ascontiguousarray(ids, dtype=np.uint32)
        self._check(self._fn("set_byzantine")(self._h, int(a.size), a.ctypes.data if a.size else None, int(delta)))

    def anomaly_flags(self): return self._get("anomaly_flags", np.uint8)

    def byzantine_stats(self):
        s = ByzantineStats()
        self._check(self._fn("byzantine_stats")(self._h, C.byref(s)))
        return s.as_dict()

    # -- user events (Serf::user_event, serf/api.rs:241-299) ------------------------------
    def set_user_events(self, content_ids):
        a = np.ascontiguousarray(content_ids, dtype=np.uint32)
        self._ue_keep = a
        self._check(self._fn("set_user_events")(self._h, int(a.size), a.ctypes.data if a.size else None))

    def user_event(self, node, event, tick=0):
        self.inject(tick, Op.USER_EVENT, node, event)

    def event_time(self): return self._get("event_time", np.uint64)
    def user_event_seen(self, event): return self._get("user_event_seen", np.uint8, event)
    def user_event_records(self): return self._get("user_event_records", UEVENT_RECORD_DTYPE)

    def user_event_ltime(self, event):
        t = _u64()
        self._check(self._fn("user_event_ltime")(self._h, int(event), C.byref(t)))
        return t.value

    def set_user_event_content(self, names, payloads):
        """The bytes of every tracked user event — what Serf::user_event(name, payload, cc) carries — after set_user_events with
        as many events.  From then on every push-pull message (wire_local_state_range) carries the node's event ring."""
        if len(names) != len(payloads):
            raise ValueError("one name and one payload per tracked event")
        raw = [x.encode() if isinstance(x, str) else bytes(x) for x in list(names) + list(payloads)]
        bufs = [C.create_string_buffer(b, max(1, len(b))) for b in raw]
        n = len(names)
        ptrs = [C.addressof(b) for b in bufs]
        lens = [len(b) for b in raw]
        self._check(self._lib.serfsim_set_user_event_content(self._h, n, (_vp * n)(*ptrs[:n]), (C.c_size_t * n)(*lens[:n]),
                                                             (_vp * n)(*ptrs[n:]), (C.c_size_t * n)(*lens[n:])))

    def wire_local_state_range(self, first=0, count=None):
        """SerfDelegate::local_state of the shard-local nodes [first, first + count), encoded on the device:
        (uint8 bytes, uint64 offsets[count + 1]); message i is bytes[offsets[i]:offsets[i + 1]]."""
        count = self.count - first if count is None else count
        off = np.zeros(count + 1, np.uint64)
        tot = C.c_size_t()
        f = self._lib.serfsim_wire_local_state_range
        f(self._h, first, count, None, 0, off.ctypes.data, C.byref(tot))                 # sizing call: reports the total
        out = np.empty(max(1, tot.value), np.uint8)
        self._check(f(self._h, first, count, out.ctypes.data, out.size, off.ctypes.data, C.byref(tot)))
        return out[:tot.value], off

    def wire_decode_events(self, buf, offsets):
        """The event rings of n push-pull messages back to the simulator's form, on the device: (event_ltime uint64[n],
        seen uint32[n] — bit e: tracked event e is in the ring —, unmatched uint32[n] — events matching no tracked event)."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        if offsets.ndim != 1 or offsets.size == 0 or offsets.size > 2**32:
            raise ValueError("offsets must be a 1-D array of n + 1 entries, 0 <= n < 2**32")
        if int(offsets[-1]) > buf.size:
            raise ValueError(f"offsets[-1] = {int(offsets[-1])} is past the end of the {buf.size}-byte buffer")
        n = offsets.size - 1
        ev, seen, um = np.zeros(n, np.uint64), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        self._check(self._lib.serfsim_wire_decode_events_batch(self._h, buf.ctypes.data, offsets.ctypes.data, n, ev.ctypes.data,
                                                               seen.ctypes.data, um.ctypes.data))
        return ev, seen, um

    def user_event_stats(self):
        s = UserEventStats()
        self._check(self._fn("user_event_stats")(self._h, C.byref(s)))
        return s.as_dict()

    def stats(self):                                                                           # Serf::stats
        s = Stats()
        self._check(self._fn("stats")(self._h, C.byref(s)))
        return s.as_dict()

    def tick_trace(self, first=0, n=None):
        if n is None:
            n = self.stats()["tick"] - first
        out = np.zeros(n, dtype=TRACE_DTYPE)
        if n:
            self._check(self._fn("tick_trace")(self._h, int(first), int(n), out.ctypes.data))
        return out

    def state_hash(self):
        h = _u64()
        self._check(self._fn("state_hash")(self._h, C.byref(h)))
        return h.value

    # -- product-only hooks -------------------------------------------------------------
    def last_step_device_ms(self):
        ms, n = C.c_double(), _u64()
        self._check(self._lib.serfsim_last_step_device_ms(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def set_tick_timing(self, enabled=True):
        self._check(self._lib.serfsim_set_tick_timing(self._h, int(enabled)))

    def tick_times_ms(self, first=0, n=None):
        if n is None:
            n = self.stats()["tick"] - first
        out = np.zeros(n, dtype=np.float32)
        if n:
            self._check(self._lib.serfsim_tick_times(self._h, int(first), int(n), out.ctypes.data))
        return out

    def tick_view_kinds(self, first=0, n=None):
        """[n, slots, 3] messages (leave, join, memberlist) each view sent per tick, counted by the per-view passes (zero in ticks without)."""
        if n is None:
            n = self.stats()["tick"] - first
        out = np.zeros((n, self.slots, 3), dtype=np.uint32)
        if n:
            self._check(self._lib.serfsim_tick_view_kinds(self._h, int(first), int(n), out.ctypes.data))
        return out

    def set_event_callback(self, fn):
        """fn(tick, type, ids) — batched EventDelegate (serf/delegate.rs:557-582)."""
        def tramp(_user, tick, ty, ids, n):
            fn(tick, ty, [ids[i] for i in range(n)])
        cb = EVENT_CB(tramp)
        self._keep.append(cb)
        self._check(self._lib.serfsim_set_event_cb(self._h, cb, None))

    def connect(self, all_gather_bytes, barrier, allreduce_u64):
        """Multi-GPU wiring: exchange CUDA-IPC window handles and install the host collectives.
        all_gather_bytes(bytes) -> list[bytes] in rank order; barrier(); allreduce_u64(np.ndarray) in place."""
        def _bar(_u):
            barrier()

        def _ar(_u, buf, n):
            arr = np.ctypeslib.as_array(buf, shape=(n,))
            allreduce_u64(arr)
        b, a = BARRIER_FN(_bar), ALLREDUCE_FN(_ar)
        self._keep += [b, a]
        self._check(self._lib.serfsim_comm_set_hooks(self._h, b, a, None))
        size = self._lib.serfsim_comm_blob_size()
        blob = C.create_string_buffer(size)
        self._check(self._lib.serfsim_comm_export(self._h, blob))
        blobs = b"".join(all_gather_bytes(blob.raw))
        assert len(blobs) == size * self.cfg.world_size
        self._check(self._lib.serfsim_comm_connect(self._h, blobs))


    def connect_loopback(self):
        """Profiling aid: a world_size = W handle (rank 0) that exchanges with itself — the per-GPU work of a W-rank run on
        one GPU (tools/loopback_profile.py).  Its simulation results are meaningless."""
        self._check(self._lib.serfsim_comm_loopback(self._h))


# ---- synthetic topologies (BASELINE.json configs) -------------------------------------
def bind_thread_near_gpu(cuda_index):
    """Pin the calling thread (and the threads it creates afterwards: the CUDA runtime's workers, torch's pinned-memory
    allocations by first touch) to the CPUs that share a NUMA node with GPU `cuda_index`.  A driver thread on the other socket
    pays the inter-socket hop on every launch and lands its pinned result buffers in far memory; two runs of the same bench
    differed by 15 % end to end depending on where the scheduler had put the process.  Returns the CPU set, or None when NVML
    (nvidia-ml-py) or the affinity call is not available — nothing is changed then."""
    import os
    try:
        import pynvml
        import torch
        pynvml.nvmlInit()
        uuid = str(torch.cuda.get_device_properties(cuda_index).uuid)
        try:
            h = pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + uuid) if not uuid.startswith("GPU-") else uuid)
        except Exception:
            h = pynvml.nvmlDeviceGetHandleByIndex(cuda_index)
        words = pynvml.nvmlDeviceGetCpuAffinity(h, (os.cpu_count() + 63) // 64)
        cpus = {64 * i + b for i, w in enumerate(words) for b in range(64) if (int(w) >> b) & 1} & os.sched_getaffinity(0)
        if not cpus:
            return None
        os.sched_setaffinity(0, cpus)
        return cpus
    except Exception:
        return None


def full_mesh_graph(n):
    """Every node may gossip with every other node (config 1: 256-node full mesh)."""
    col = np.empty((n, n - 1), dtype=np.uint32)
    ar = np.arange(n, dtype=np.uint32)
    for v in range(n):
        col[v, :v] = ar[:v]
        col[v, v:] = ar[v + 1:]
    row_ptr = np.arange(n + 1, dtype=np.uint64) * np.uint64(n - 1)
    return row_ptr, col.reshape(-1)


def random_regular_graph(n, degree, seed):
    """Each node draws `degree` out-neighbours uniformly (≠ itself; repeats are rare and harmless)."""
    rng = np.random.Generator(np.random.Philox(seed))
    col = rng.integers(0, n - 1, size=(n, degree), dtype=np.uint32)
    col += (col >= np.arange(n, dtype=np.uint32)[:, None]).astype(np.uint32)      # skip self
    row_ptr = np.arange(n + 1, dtype=np.uint64) * np.uint64(degree)
    return row_ptr, col.reshape(-1)


def small_world_graph(n, k, beta, seed):
    """Watts–Strogatz ring lattice (k nearest neighbours) with rewiring probability beta."""
    rng = np.random.Generator(np.random.Philox(seed))
    offs = np.concatenate([np.arange(1, k // 2 + 1), -np.arange(1, k // 2 + 1)]).astype(np.int64)
    col = (np.arange(n, dtype=np.int64)[:, None] + offs[None, :]) % n
    rew = rng.random(col.shape) < beta
    rnd = rng.integers(0, n - 1, size=col.shape, dtype=np.int64)
    rnd += (rnd >= np.arange(n, dtype=np.int64)[:, None])
    col = np.where(rew, rnd, col).astype(np.uint32)
    row_ptr = np.arange(n + 1, dtype=np.uint64) * np.uint64(len(offs))
    return row_ptr, col.reshape(-1)
