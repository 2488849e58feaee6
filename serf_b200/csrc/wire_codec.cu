// wire_codec.cu — serf's wire format behind the C ABI (SURVEY §8f row 4; layout and citations in wire.cuh).
//
// Single messages (Join, Leave, PushPull, with the message envelope) are encoded / decoded on the host — they are a few dozen
// bytes.  The bulk job is SerfDelegate::local_state (serf/delegate.rs:386-425): the push-pull message of a node lists every
// member it knows; producing it for all virtual nodes of a shard is an O(N·R) variable-length byte job, done on the device in
// three kernels: encoded lengths → exclusive scan → byte emission (one thread per node for the membership part, the warp for
// the event ring a content table adds — up to ~4 KB per node).  The inverse batches (decode n messages into per-node arrays,
// or their rings into seen masks) are the device half of merge_remote_state's parsing.
#include <cstring>
#include <string>
#include <vector>

#include "../../include/serfsim.h"
#include "owned.cuh"
#include "tick_kernel.cuh"
#include "wire.cuh"

using namespace sfs;
namespace w = sfs::wire;

struct serfsim;                                   // serfsim.cu
namespace sfs {
struct WireView { const uint4* rec; const u32* qword; const u64* node_state; const uint4* ue_state; const u32* subj; u32 n_local, stride, R; cudaStream_t stream; wire::UeWire ue; };
int serfsim_wire_view(const serfsim* h, WireView* out);          // serfsim.cu: the device arrays a batch encode reads
}

namespace {

int werr(int rc) {
  switch (rc) {
    case w::E_TRUNCATED: return serfsim_fail(SERFSIM_E_INVAL, "wire: truncated message");
    case w::E_VARINT: return serfsim_fail(SERFSIM_E_INVAL, "wire: varint longer than 64 bits");
    case w::E_DUPLICATE: return serfsim_fail(SERFSIM_E_INVAL, "wire: duplicate field");
    case w::E_MISSING: return serfsim_fail(SERFSIM_E_INVAL, "wire: missing field");
    case w::E_WIRE_TYPE: return serfsim_fail(SERFSIM_E_INVAL, "wire: unknown wire type");
    case w::E_CAPACITY: return serfsim_fail(SERFSIM_E_INVAL, "wire: output capacity too small");
    case w::E_TYPE: return serfsim_fail(SERFSIM_E_INVAL, "wire: not a message of the requested type");
    default: return serfsim_fail(SERFSIM_E_INVAL, "wire: malformed message");
  }
}

// One node's local_state (serf/delegate.rs:386-425) from its views: the member table of a virtual node holds the tracked
// subjects it knows; left_members lists those it has as Left; the event clock comes from the user-event record (1 when user
// events are off — a fresh node, serf/base.rs:198-200), the query clock is not modelled (1).  With a content table the node's
// event ring is attached (below); without one no events are.
struct NodeState { u64 ltime, event_ltime; u32 known, left, seen; };   // bit s of known / left: subject s; seen: tracked events

// The ring of a node (EventCore.buffer, serf/base.rs:193) from its `seen` mask: one UserEvents per occupied slot, slots by
// ascending ring index (ltime % 512) as PushPullMessageBorrow walks the buffer (push_pull.rs:566-577, empty slots skipped),
// the slot's ltime being the ltime of its events (cluster runs keep one per slot, DESIGN §8.3).  Inside a slot the packed
// record keeps no arrival order: events by ascending tracked index.  f(slot_mask, ltime, entry_bytes) per slot, in order.
template <class F>
__device__ __forceinline__ void for_each_ring_slot(u32 seen, const u32* lt, const u32* off, F&& f) {
  while (seen) {
    u32 lead = 0, key = 0xffffffffu;
    for (u32 e = 0; e < w::UE_TABLE_MAX; ++e)
      if ((seen >> e) & 1u) { const u32 k = ((lt[e] % 512u) << 4) | e; if (k < key) { key = k; lead = e; } }
    u32 slot = 0, bytes = 0;
    for (u32 e = 0; e < w::UE_TABLE_MAX; ++e)
      if (((seen >> e) & 1u) && lt[e] % 512u == lt[lead] % 512u) { slot |= 1u << e; bytes += off[e + 1] - off[e]; }
    f(slot, lt[lead], bytes);
    seen &= ~slot;
  }
}
__device__ __forceinline__ u32 ring_len(u32 seen, const u32* lt, const u32* off) {
  u32 len = 0;
  for_each_ring_slot(seen, lt, off, [&](u32, u32 L, u32 bytes) { len += w::pp_events_entry_len(L, bytes); });
  return len;
}

// lt: the tracked events' Lamport times (nullptr: no content table)
__device__ __forceinline__ u32 pp_payload_len(const WireView& v, u32 vl, const u32* lt, NodeState* st_out, u64* sts) {
  NodeState st{};
  st.ltime = nw_clock(v.node_state[vl]);
  st.event_ltime = v.ue_state ? v.ue_state[vl].x : 1u;
  st.seen = lt ? (v.ue_state[vl].y & ((1u << v.ue.n) - 1u)) : 0u;
  u32 len = 1 + w::varint_len(st.ltime);
  for (u32 s = 0; s < v.R; ++s) {
    Rec r;
    unpack(load_rec(v.rec, (size_t)s * v.stride + vl), r);
    if (!(r.flags & FLAG_KNOWN)) continue;
    st.known |= 1u << s;
    if (sts) sts[s] = r.st;
    len += w::pp_status_entry_len(v.subj[s], r.st);
    if (r.status == ST_LEFT) { st.left |= 1u << s; }
  }
  for (u32 s = 0; s < v.R; ++s) if ((st.left >> s) & 1u) len += w::pp_left_entry_len(v.subj[s]);
  len += 1 + w::varint_len(st.event_ltime) + 1 + w::varint_len(1);
  if (st.seen) len += ring_len(st.seen, lt, v.ue.off);
  *st_out = st;
  return len;
}
// Nodes [first, first + count) of the shard; lens / offsets / out are relative to the range.
__global__ void pp_len_kernel(WireView v, u32 first, u32 count, u64* lens) {
  __shared__ u32 s_lt[w::UE_TABLE_MAX];
  if (v.ue.n) {
    if (threadIdx.x < w::UE_TABLE_MAX) s_lt[threadIdx.x] = threadIdx.x < v.ue.n ? v.ue.ltime[threadIdx.x] : 0u;
    __syncthreads();
  }
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  NodeState st;
  lens[i] = w::envelope_len(pp_payload_len(v, first + i, v.ue.n ? s_lt : nullptr, &st, nullptr));
}
// single-CTA exclusive scan over n u64 lengths (n ≤ a few 10 M: 1024 threads, a chunk each, then the chunk totals)
__global__ void __launch_bounds__(1024) pp_scan_kernel(const u64* lens, u64* offsets, u32 n) {
  __shared__ u64 part[1024];
  const u32 per = (n + 1023) / 1024, b = threadIdx.x * per, e = min(n, b + per);
  u64 s = 0;
  for (u32 i = b; i < e; ++i) s += lens[i];
  part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) { u64 acc = 0; for (int i = 0; i < 1024; ++i) { const u64 t = part[i]; part[i] = acc; acc += t; } offsets[n] = acc; }
  __syncthreads();
  u64 acc = part[threadIdx.x];
  for (u32 i = b; i < e; ++i) { offsets[i] = acc; acc += lens[i]; }
}
// One thread per node writes the membership part and the clocks; the event ring — up to 8 entries of ≤ 521 bytes, identical
// for every node that holds the event — is copied by the whole warp, node after node, from the CTA's shared-memory copy of
// the content table.
constexpr u32 EMIT_THREADS = 256;
__global__ void __launch_bounds__(EMIT_THREADS) pp_emit_kernel(WireView v, u32 first, u32 count, const u64* offsets, u8* out, u64 cap) {
  __shared__ __align__(16) u8 s_entries[w::UE_TABLE_MAX * w::UE_ENTRY_MAX];
  __shared__ u32 s_lt[w::UE_TABLE_MAX];
  const bool events = v.ue.n != 0;
  if (events) {
    const u32 nb = v.ue.off[v.ue.n];
    for (u32 b = threadIdx.x; b < nb; b += blockDim.x) s_entries[b] = v.ue.entries[b];
    if (threadIdx.x < w::UE_TABLE_MAX) s_lt[threadIdx.x] = threadIdx.x < v.ue.n ? v.ue.ltime[threadIdx.x] : 0u;
    __syncthreads();
  }
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  u32 seen = 0;
  u64 ring_at = 0;                                               // where this node's ring entries start in `out`
  if (i < count) {
    NodeState st;
    u64 sts[MAX_SLOTS];
    const u32 pl = pp_payload_len(v, first + i, events ? s_lt : nullptr, &st, sts);
    if (offsets[i] + w::envelope_len(pl) <= cap) {               // else the host reports the shortfall from offsets[count]
      u8* p = out + offsets[i];
      u32 o = 0;
      p[o++] = w::MSG_PUSH_PULL; o += w::varint_put(p + o, pl);                           // message.rs:397-428
      p[o++] = w::PP_LTIME; o += w::varint_put(p + o, st.ltime);                          // push_pull.rs:383-386
      for (u32 s = 0; s < v.R; ++s) if ((st.known >> s) & 1u) o += w::put_pp_status_entry(p + o, v.subj[s], sts[s]);   // :388-398
      for (u32 s = 0; s < v.R; ++s) if ((st.left >> s) & 1u) { p[o++] = w::PP_LEFT; o += w::varint_put(p + o, v.subj[s]); }   // :400-411
      p[o++] = w::PP_EVENT_LTIME; o += w::varint_put(p + o, st.event_ltime);              // :413-416
      if (st.seen) { seen = st.seen; ring_at = offsets[i] + o; o += ring_len(st.seen, s_lt, v.ue.off); }   // :418-428, by the warp
      p[o++] = w::PP_QUERY_LTIME; o += w::varint_put(p + o, 1);                           // :430-433
    }
  }
  if (!events) return;
  const u32 lane = threadIdx.x & 31u;
  u32 todo = __ballot_sync(0xffffffffu, seen != 0);
  while (todo) {
    const int j = __ffs((int)todo) - 1;
    todo &= todo - 1;
    const u32 sj = __shfl_sync(0xffffffffu, seen, j);
    const u32 lo = __shfl_sync(0xffffffffu, (u32)ring_at, j), hi = __shfl_sync(0xffffffffu, (u32)(ring_at >> 32), j);
    u8* p = out + (((u64)hi << 32) | lo);
    for_each_ring_slot(sj, s_lt, v.ue.off, [&](u32 slot, u32 L, u32 bytes) {
      if (lane == 0) w::put_pp_events_head(p, L, bytes);
      p += 1 + w::varint_len(w::ues_body_len(L, bytes)) + 1 + w::varint_len(L);
      for (u32 e = 0; e < v.ue.n; ++e) {
        if (!((slot >> e) & 1u)) continue;
        const u32 b0 = v.ue.off[e], nb = v.ue.off[e + 1] - b0;
        for (u32 b = lane; b < nb; b += 32) p[b] = s_entries[b0 + b];
        p += nb;
      }
    });
  }
}

// PushPullMessageRef::decode (push_pull.rs:175-317) on one payload, arrays bounded by `cap` entries (store == false: status
// and left entries are checked and counted, not stored).  on_events(entry body, its length, its offset in p)
// is called for every `events` entry and returns OK or an error.
template <class OnEvents>
__host__ __device__ int pp_decode_payload_ev(const u8* p, size_t len, u64* ltime, u64* event_ltime, u64* query_ltime, u64* ids, u64* sts, u32 cap, u32* n_status,
                                             u64* left, u32 left_cap, u32* n_left, bool store, OnEvents&& on_events) {
  size_t o = 0;
  bool h_lt = false, h_ev = false, h_q = false;
  u32 ns = 0, nl = 0;
  while (o < len) {
    const u8 b = p[o];
    if (b == w::PP_LTIME || b == w::PP_EVENT_LTIME || b == w::PP_QUERY_LTIME) {
      bool& have = b == w::PP_LTIME ? h_lt : b == w::PP_EVENT_LTIME ? h_ev : h_q;
      if (have) return w::E_DUPLICATE;
      u64 v;
      const int r = w::varint_get(p + o + 1, len - o - 1, &v);
      if (r < 0) return r;
      *(b == w::PP_LTIME ? ltime : b == w::PP_EVENT_LTIME ? event_ltime : query_ltime) = v;
      have = true; o += 1 + r;
    } else if (b == w::PP_STATUS) {                          // one (id, status_time) tuple, length-delimited
      u64 tl;
      const int r = w::varint_get(p + o + 1, len - o - 1, &tl);
      if (r < 0) return r;
      if ((u64)(len - o - 1 - r) < tl) return w::E_TRUNCATED;
      const u8* t = p + o + 1 + r;
      size_t to = 0;
      u64 id = 0, st = 0; bool hk = false, hv = false;
      while (to < tl) {
        if (t[to] == w::TUPLE_KEY || t[to] == w::TUPLE_VALUE) {
          u64 v;
          const int r2 = w::varint_get(t + to + 1, (size_t)tl - to - 1, &v);
          if (r2 < 0) return r2;
          if (t[to] == w::TUPLE_KEY) { id = v; hk = true; } else { st = v; hv = true; }
          to += 1 + r2;
        } else {
          const long s = w::skip_field(t + to, (size_t)tl - to);
          if (s < 0) return (int)s;
          to += (size_t)s;
        }
      }
      if (!hk || !hv) return w::E_MISSING;
      if (store) {
        if (ns >= cap) return w::E_CAPACITY;
        ids[ns] = id; sts[ns] = st;
      }
      ++ns;
      o += 1 + r + (size_t)tl;
    } else if (b == w::PP_LEFT) {
      u64 v;
      const int r = w::varint_get(p + o + 1, len - o - 1, &v);
      if (r < 0) return r;
      if (store) {
        if (nl >= left_cap) return w::E_CAPACITY;
        left[nl] = v;
      }
      ++nl;
      o += 1 + r;
    } else if (b == w::PP_EVENTS) {
      u32 off, n;
      const int r = w::get_len_delim(p + o + 1, len - o - 1, &off, &n);
      if (r < 0) return r;
      const int rc = on_events(p + o + 1 + off, (size_t)n, (u32)(o + 1 + off));
      if (rc) return rc;
      o += 1 + r;
    } else {
      const long s = w::skip_field(p + o, len - o);
      if (s < 0) return (int)s;
      o += (size_t)s;
    }
  }
  if (!h_lt || !h_ev || !h_q) return w::E_MISSING;            // push_pull.rs:292-316
  *n_status = ns; *n_left = nl;
  return w::OK;
}
// The membership path: `events` entries are counted and skipped.
__host__ __device__ int pp_decode_payload(const u8* p, size_t len, u64* ltime, u64* event_ltime, u64* query_ltime, u64* ids, u64* sts, u32 cap, u32* n_status,
                                          u64* left, u32 left_cap, u32* n_left, u32* n_events) {
  u32 ne = 0;
  const int rc = pp_decode_payload_ev(p, len, ltime, event_ltime, query_ltime, ids, sts, cap, n_status, left, left_cap, n_left, true,
                                      [&](const u8*, size_t, u32) { ++ne; return (int)w::OK; });
  if (rc == w::OK && n_events) *n_events = ne;
  return rc;
}
__global__ void pp_decode_kernel(const u8* buf, const u64* offsets, u32 n, u32 cap, u64* ltime, u64* ids, u64* sts, u32* n_status, u32* left_mask_err) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u8* m = buf + offsets[i];
  const size_t len = (size_t)(offsets[i + 1] - offsets[i]);
  u8 type = 0; size_t po = 0, pl = 0;
  int rc = w::open_envelope(m, len, &type, &po, &pl);
  if (rc == w::OK && type != w::MSG_PUSH_PULL) rc = w::E_TYPE;
  u64 ev, q, left[MAX_SLOTS];
  u32 ns = 0, nl = 0;
  if (rc == w::OK) rc = pp_decode_payload(m + po, pl, ltime + i, &ev, &q, ids + (size_t)i * cap, sts + (size_t)i * cap, cap, &ns, left, MAX_SLOTS, &nl, nullptr);
  n_status[i] = rc == w::OK ? ns : 0;
  left_mask_err[i] = rc == w::OK ? nl : 0x80000000u | (u32)(-rc);
}

// The rings back to the simulator's form: message i → its event clock, the mask of tracked events its ring holds (tracked event
// e matches a UserEvent with e's name and payload bytes in an entry whose ltime is e's Lamport time; equal content and equal
// ltime → the lowest index), and the number of events that match no tracked event.  One thread per message.
__global__ void pp_events_decode_kernel(const u8* buf, const u64* offsets, u32 n, w::UeWire ue, u64* event_ltime, u32* seen, u32* unmatched, u32* err) {
  __shared__ __align__(16) u8 s_entries[w::UE_TABLE_MAX * w::UE_ENTRY_MAX];
  __shared__ u32 s_lt[w::UE_TABLE_MAX];
  for (u32 b = threadIdx.x; b < ue.off[ue.n]; b += blockDim.x) s_entries[b] = ue.entries[b];
  if (threadIdx.x < w::UE_TABLE_MAX) s_lt[threadIdx.x] = threadIdx.x < ue.n ? ue.ltime[threadIdx.x] : 0u;
  __syncthreads();
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u8* m = buf + offsets[i];
  const size_t len = (size_t)(offsets[i + 1] - offsets[i]);
  u8 type = 0; size_t po = 0, pl = 0;
  int rc = w::open_envelope(m, len, &type, &po, &pl);
  if (rc == w::OK && type != w::MSG_PUSH_PULL) rc = w::E_TYPE;
  u64 lt = 0, ev = 0, q = 0;
  u32 ns = 0, nl = 0, mask = 0, um = 0;
  auto same = [&](const u8* p, u32 off, u32 n_, u32 ref_off, u32 ref_n) {
    if (n_ != ref_n) return false;
    for (u32 k = 0; k < n_; ++k) if (p[off + k] != s_entries[ref_off + k]) return false;
    return true;
  };
  if (rc == w::OK)
    rc = pp_decode_payload_ev(m + po, pl, &lt, &ev, &q, nullptr, nullptr, 0, &ns, nullptr, 0, &nl, false, [&](const u8* body, size_t blen, u32) {
      u64 L = 0; u32 ne = 0;
      return w::walk_user_events(body, blen, 0, &L, &ne, [&](const w::EventBytes& eb) {
        u32 e = 0;
        for (; e < ue.n; ++e)
          if (s_lt[e] && (u64)s_lt[e] == L && same(body, eb.name_off, eb.name_len, ue.bytes[e].name_off, ue.bytes[e].name_len) &&
              same(body, eb.pay_off, eb.pay_len, ue.bytes[e].pay_off, ue.bytes[e].pay_len)) break;
        if (e < ue.n) mask |= 1u << e; else ++um;
        return (int)w::OK;
      });
    });
  event_ltime[i] = rc == w::OK ? ev : 0;
  seen[i] = rc == w::OK ? mask : 0;
  unmatched[i] = rc == w::OK ? um : 0;
  err[i] = rc == w::OK ? 0u : 0x80000000u | (u32)(-rc);
}

// PushPull with or without a ring (push_pull.rs:483-587); *len = the needed size, also on failure.
int encode_pp(const serfsim_wire_push_pull_t* m, const serfsim_wire_user_events_t* ring, u32 n_ring, uint8_t* buf, size_t cap, size_t* len) {
  if (!m || !len || (m->n_status && (!m->status_ids || !m->status_ltimes)) || (m->n_left && !m->left_ids) || (n_ring && !ring)) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
  std::vector<u64> entries(n_ring, 0);                     // bytes of the events entries of ring entry k
  for (u32 k = 0; k < n_ring; ++k) {
    if (ring[k].n_events && !ring[k].events) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
    for (u32 j = 0; j < ring[k].n_events; ++j) {
      const serfsim_wire_event_t& e = ring[k].events[j];
      if ((e.name_len && !e.name) || (e.payload_len && !e.payload)) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
      if (e.name_len > 0xffffffu || e.payload_len > 0xffffffu) return serfsim_fail(SERFSIM_E_INVAL, "wire: message too large");
      entries[k] += w::ues_event_entry_len((u32)e.name_len, (u32)e.payload_len);
    }
    if (entries[k] > 0x7fffffffull) return serfsim_fail(SERFSIM_E_INVAL, "wire: message too large");
  }
  size_t pl = 1 + w::varint_len(m->ltime);
  for (u32 i = 0; i < m->n_status; ++i) pl += w::pp_status_entry_len(m->status_ids[i], m->status_ltimes[i]);
  for (u32 i = 0; i < m->n_left; ++i) pl += w::pp_left_entry_len(m->left_ids[i]);
  pl += 1 + w::varint_len(m->event_ltime) + 1 + w::varint_len(m->query_ltime);
  for (u32 k = 0; k < n_ring; ++k) pl += w::pp_events_entry_len(ring[k].ltime, entries[k]);
  if (pl > 0xffffffffull) return serfsim_fail(SERFSIM_E_INVAL, "wire: message too large");      // EncodeError::TooLarge, message.rs:410-412
  const size_t need = 1 + w::varint_len(pl) + pl;
  *len = need;
  if (!buf || cap < need) return werr(w::E_CAPACITY);
  size_t o = 0;
  buf[o++] = w::MSG_PUSH_PULL; o += w::varint_put(buf + o, pl);
  buf[o++] = w::PP_LTIME; o += w::varint_put(buf + o, m->ltime);
  for (u32 i = 0; i < m->n_status; ++i) o += w::put_pp_status_entry(buf + o, m->status_ids[i], m->status_ltimes[i]);
  for (u32 i = 0; i < m->n_left; ++i) { buf[o++] = w::PP_LEFT; o += w::varint_put(buf + o, m->left_ids[i]); }
  buf[o++] = w::PP_EVENT_LTIME; o += w::varint_put(buf + o, m->event_ltime);
  for (u32 k = 0; k < n_ring; ++k) {                       // push_pull.rs:566-577: UserEvents{ltime, events}, length-delimited
    o += w::put_pp_events_head(buf + o, ring[k].ltime, entries[k]);
    for (u32 j = 0; j < ring[k].n_events; ++j) {           // user_events.rs encode: [events byte][UserEvent, length-delimited]
      const serfsim_wire_event_t& e = ring[k].events[j];
      const u32 nl = (u32)e.name_len, pyl = (u32)e.payload_len;
      buf[o++] = w::UES_EVENT; o += w::varint_put(buf + o, w::user_event_len(nl, pyl));
      o += w::put_user_event(buf + o, e.name, nl, e.payload, pyl);
    }
  }
  buf[o++] = w::PP_QUERY_LTIME; o += w::varint_put(buf + o, m->query_ltime);
  return o == need ? 0 : serfsim_fail(SERFSIM_E_INVAL, "wire: internal length mismatch");
}

// The batch decoders copy offsets[n] bytes of `buf` to the device and give message i the slice [offsets[i], offsets[i + 1]):
// non-decreasing offsets keep every slice inside those bytes.  Checked before anything is allocated or launched.
int check_batch_offsets(const uint64_t* offsets, u32 n) {
  for (u32 i = 0; i < n; ++i)
    if (offsets[i] > offsets[i + 1])
      return serfsim_fail(SERFSIM_E_INVAL, (std::string("wire: offsets[") + std::to_string(i) + "] > offsets[" + std::to_string(i + 1) + "]: message " +
                                            std::to_string(i) + " would end before it starts").c_str());
  return 0;
}

}  // namespace

#pragma GCC visibility push(default)
extern "C" {

size_t serfsim_wire_encoded_len_intent(const serfsim_wire_intent_t* m) {
  if (!m) return 0;
  return w::envelope_len(m->type == SERFSIM_WIRE_JOIN ? w::join_payload_len(m->ltime, m->id) : w::leave_payload_len(m->ltime, m->id, m->prune != 0));
}

int serfsim_wire_encode_intent(const serfsim_wire_intent_t* m, uint8_t* buf, size_t cap, size_t* len) {
  if (!m || !buf || !len) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
  if (m->type != SERFSIM_WIRE_JOIN && m->type != SERFSIM_WIRE_LEAVE) return serfsim_fail(SERFSIM_E_INVAL, "wire: intent type must be SERFSIM_WIRE_JOIN or SERFSIM_WIRE_LEAVE");
  const size_t need = serfsim_wire_encoded_len_intent(m);
  *len = need;
  if (cap < need) return werr(w::E_CAPACITY);                 // EncodeError::insufficient_buffer: the needed size is reported in *len
  const u32 n = m->type == SERFSIM_WIRE_JOIN ? w::put_join(buf, m->ltime, m->id) : w::put_leave(buf, m->ltime, m->id, m->prune != 0);
  return n == need ? 0 : serfsim_fail(SERFSIM_E_INVAL, "wire: internal length mismatch");
}

int serfsim_wire_message_type(const uint8_t* buf, size_t len, uint32_t* type) {
  if (!buf || !type) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
  u8 t = 0; size_t po = 0, pl = 0;
  const int rc = w::open_envelope(buf, len, &t, &po, &pl);
  if (rc) return werr(rc);
  *type = t == w::MSG_LEAVE ? SERFSIM_WIRE_LEAVE : t == w::MSG_JOIN ? SERFSIM_WIRE_JOIN : t == w::MSG_PUSH_PULL ? SERFSIM_WIRE_PUSH_PULL : SERFSIM_WIRE_USER_EVENT;
  return 0;
}

int serfsim_wire_decode_intent(const uint8_t* buf, size_t len, serfsim_wire_intent_t* out) {
  if (!buf || !out) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
  u8 t = 0; size_t po = 0, pl = 0;
  int rc = w::open_envelope(buf, len, &t, &po, &pl);
  if (rc) return werr(rc);
  if (t != w::MSG_JOIN && t != w::MSG_LEAVE) return werr(w::E_TYPE);
  w::Intent in{};
  rc = w::get_intent(buf + po, pl, t == w::MSG_LEAVE, &in);
  if (rc) return werr(rc);
  out->type = t == w::MSG_LEAVE ? SERFSIM_WIRE_LEAVE : SERFSIM_WIRE_JOIN; out->prune = in.prune ? 1u : 0u; out->ltime = in.ltime; out->id = in.id;
  return 0;
}

int serfsim_wire_encode_push_pull(const serfsim_wire_push_pull_t* m, uint8_t* buf, size_t cap, size_t* len) {
  return encode_pp(m, nullptr, 0, buf, cap, len);
}

int serfsim_wire_decode_push_pull(const uint8_t* buf, size_t len, serfsim_wire_push_pull_t* out) {
  if (!buf || !out) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
  u8 t = 0; size_t po = 0, pl = 0;
  int rc = w::open_envelope(buf, len, &t, &po, &pl);
  if (rc) return werr(rc);
  if (t != w::MSG_PUSH_PULL) return werr(w::E_TYPE);
  u32 ns = 0, nl = 0, ne = 0;
  rc = pp_decode_payload(buf + po, pl, &out->ltime, &out->event_ltime, &out->query_ltime, out->status_ids, out->status_ltimes, out->n_status, &ns,
                         out->left_ids, out->n_left, &nl, &ne);
  if (rc) return werr(rc);
  out->n_status = ns; out->n_left = nl; out->n_events_skipped = ne;
  return 0;
}

// SerfDelegate::local_state of the shard-local nodes [first, first + count), on the device.  offsets: [count + 1] byte offsets
// into `out` (offsets[0] = 0, offsets[count] = total).  With out == NULL or cap too small only the offsets are produced and
// SERFSIM_E_INVAL is returned with *total set, so that the caller can size the buffer.
int serfsim_wire_local_state_range(serfsim_t* h, uint32_t first, uint32_t count, uint8_t* out, size_t cap, uint64_t* offsets, size_t* total) {
  if (!h || !offsets || !total) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
  WireView v{};
  int rc = serfsim_wire_view(h, &v);
  if (rc) return rc;
  if (first > v.n_local || count > v.n_local - first) return serfsim_fail(SERFSIM_E_INVAL, "wire: node range outside the shard");
  const u32 n = count;
  DevArray<u64> d_len, d_off;
  DevArray<u8> d_out;
  CU(d_len.alloc((size_t)n + 1)); CU(d_off.alloc((size_t)n + 1));
  if (n) SFS_LAUNCH((n + 255) / 256, 256, 0, v.stream, pp_len_kernel)(v, first, n, d_len.get());
  SFS_LAUNCH(1, 1024, 0, v.stream, pp_scan_kernel)(d_len.get(), d_off.get(), n);
  CU(cudaMemcpyAsync(offsets, d_off, d_off.bytes(), cudaMemcpyDeviceToHost, v.stream));
  CU(cudaStreamSynchronize(v.stream));
  *total = (size_t)offsets[n];
  if (!out || cap < *total) return werr(w::E_CAPACITY);
  CU(d_out.alloc(*total ? *total : 1));
  if (n) SFS_LAUNCH((n + EMIT_THREADS - 1) / EMIT_THREADS, EMIT_THREADS, 0, v.stream, pp_emit_kernel)(v, first, n, d_off.get(), d_out.get(), (u64)*total);
  CU(cudaMemcpyAsync(out, d_out, *total, cudaMemcpyDeviceToHost, v.stream));
  CU(cudaStreamSynchronize(v.stream));
  CU(cudaGetLastError());
  return 0;
}

// Every node of the shard: the range over the whole shard.
int serfsim_wire_local_state_batch(serfsim_t* h, uint8_t* out, size_t cap, uint64_t* offsets, size_t* total) {
  if (!h || !offsets || !total) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
  WireView v{};
  int rc = serfsim_wire_view(h, &v);
  if (rc) return rc;
  return serfsim_wire_local_state_range(h, 0, v.n_local, out, cap, offsets, total);
}

// The inverse batch on the device: n push-pull messages (concatenated, offsets[n + 1]) → per message the Lamport clock, up to
// `cap` (id, status_time) entries and their count.  A malformed message fails the call (index in the error text).
int serfsim_wire_decode_batch(serfsim_t* h, const uint8_t* buf, const uint64_t* offsets, uint32_t n, uint32_t cap, uint64_t* ltime, uint64_t* ids, uint64_t* status_ltimes, uint32_t* n_status) {
  if (!h || !buf || !offsets || !ltime || !ids || !status_ltimes || !n_status || !cap) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
  WireView v{};
  int rc = serfsim_wire_view(h, &v);
  if (rc) return rc;
  if ((rc = check_batch_offsets(offsets, n))) return rc;
  if (!n) return 0;                                          // nothing to decode
  const size_t total = (size_t)offsets[n];
  DevArray<u8> d_buf;
  DevArray<u64> d_off, d_lt, d_ids, d_sts;
  DevArray<u32> d_ns, d_err;
  CU(d_buf.alloc(total ? total : 1)); CU(d_off.alloc((size_t)n + 1)); CU(d_lt.alloc(n));
  CU(d_ids.alloc((size_t)n * cap)); CU(d_sts.alloc((size_t)n * cap)); CU(d_ns.alloc(n)); CU(d_err.alloc(n));
  CU(cudaMemcpyAsync(d_buf, buf, total, cudaMemcpyHostToDevice, v.stream));
  CU(cudaMemcpyAsync(d_off, offsets, d_off.bytes(), cudaMemcpyHostToDevice, v.stream));
  SFS_LAUNCH((n + 127) / 128, 128, 0, v.stream, pp_decode_kernel)(d_buf.get(), d_off.get(), n, cap, d_lt.get(), d_ids.get(), d_sts.get(), d_ns.get(), d_err.get());
  std::vector<u32> err(n);
  CU(cudaMemcpyAsync(ltime, d_lt, d_lt.bytes(), cudaMemcpyDeviceToHost, v.stream));
  CU(cudaMemcpyAsync(ids, d_ids, d_ids.bytes(), cudaMemcpyDeviceToHost, v.stream));
  CU(cudaMemcpyAsync(status_ltimes, d_sts, d_sts.bytes(), cudaMemcpyDeviceToHost, v.stream));
  CU(cudaMemcpyAsync(n_status, d_ns, d_ns.bytes(), cudaMemcpyDeviceToHost, v.stream));
  CU(cudaMemcpyAsync(err.data(), d_err, d_err.bytes(), cudaMemcpyDeviceToHost, v.stream));
  CU(cudaStreamSynchronize(v.stream));
  CU(cudaGetLastError());
  for (u32 i = 0; i < n; ++i)
    if (err[i] & 0x80000000u) { werr(-(int)(err[i] & 0xffffu)); return serfsim_fail(SERFSIM_E_INVAL, (std::string("wire: message ") + std::to_string(i) + ": " + serfsim_last_error()).c_str()); }
  return 0;
}

// ---- user events ----
int serfsim_wire_encode_user_event(const serfsim_wire_user_event_t* m, uint8_t* buf, size_t cap, size_t* len) {
  if (!m || !len || (m->name_len && !m->name) || (m->payload_len && !m->payload)) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
  if (m->name_len > 0xffffffu || m->payload_len > 0xffffffu) return serfsim_fail(SERFSIM_E_INVAL, "wire: message too large");
  const u32 nl = (u32)m->name_len, pl = (u32)m->payload_len;
  const size_t need = w::envelope_len(w::uem_payload_len(m->ltime, nl, pl, m->cc != 0));
  *len = need;
  if (!buf || cap < need) return werr(w::E_CAPACITY);          // EncodeError::insufficient_buffer: the needed size is reported in *len
  const u32 n = w::put_uem(buf, m->ltime, m->name, nl, m->payload, pl, m->cc != 0);
  return n == need ? 0 : serfsim_fail(SERFSIM_E_INVAL, "wire: internal length mismatch");
}

int serfsim_wire_decode_user_event(const uint8_t* buf, size_t len, serfsim_wire_user_event_t* out) {
  if (!buf || !out) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
  u8 t = 0; size_t po = 0, pl = 0;
  int rc = w::open_envelope(buf, len, &t, &po, &pl);
  if (rc) return werr(rc);
  if (t != w::MSG_USER_EVENT) return werr(w::E_TYPE);
  u64 ltime = 0; bool cc = false; w::EventBytes eb{};
  rc = w::get_uem(buf + po, pl, (u32)po, &ltime, &eb, &cc);
  if (rc) return werr(rc);
  out->ltime = ltime; out->cc = cc ? 1u : 0u; out->pad = 0;
  out->name = eb.name_len ? buf + eb.name_off : nullptr; out->name_len = eb.name_len;
  out->payload = eb.pay_len ? buf + eb.pay_off : nullptr; out->payload_len = eb.pay_len;
  return 0;
}

int serfsim_wire_encode_push_pull_events(const serfsim_wire_push_pull_t* m, const serfsim_wire_user_events_t* ring, uint32_t n_ring, uint8_t* buf, size_t cap, size_t* len) {
  return encode_pp(m, ring, n_ring, buf, cap, len);
}

int serfsim_wire_decode_push_pull_events(const uint8_t* buf, size_t len, serfsim_wire_push_pull_t* out, serfsim_wire_user_events_t* ring, uint32_t* n_ring,
                                         serfsim_wire_event_t* events, uint32_t* n_events) {
  if (!buf || !out || !n_ring || !n_events || (*n_ring && !ring) || (*n_events && !events)) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
  u8 t = 0; size_t po = 0, pl = 0;
  int rc = w::open_envelope(buf, len, &t, &po, &pl);
  if (rc) return werr(rc);
  if (t != w::MSG_PUSH_PULL) return werr(w::E_TYPE);
  const u32 ring_cap = *n_ring, ev_cap = *n_events;
  u32 nr = 0, ne = 0, ns = 0, nl = 0;
  rc = pp_decode_payload_ev(buf + po, pl, &out->ltime, &out->event_ltime, &out->query_ltime, out->status_ids, out->status_ltimes, out->n_status, &ns,
                            out->left_ids, out->n_left, &nl, true, [&](const u8* body, size_t blen, u32 at) {
    if (nr >= ring_cap) return (int)w::E_CAPACITY;
    u64 L = 0; u32 k = 0;
    const u32 first = ne;
    const int r = w::walk_user_events(body, blen, (u32)po + at, &L, &k, [&](const w::EventBytes& eb) {
      if (ne >= ev_cap) return (int)w::E_CAPACITY;
      events[ne].name = eb.name_len ? buf + eb.name_off : nullptr; events[ne].name_len = eb.name_len;
      events[ne].payload = eb.pay_len ? buf + eb.pay_off : nullptr; events[ne].payload_len = eb.pay_len;
      ++ne;
      return (int)w::OK;
    });
    if (r) return r;
    ring[nr].ltime = L; ring[nr].n_events = k; ring[nr].pad = 0; ring[nr].events = k ? events + first : nullptr;
    ++nr;
    return (int)w::OK;
  });
  if (rc) return werr(rc);
  out->n_status = ns; out->n_left = nl; out->n_events_skipped = 0;
  *n_ring = nr; *n_events = ne;
  return 0;
}

// The rings of n push-pull messages back to the simulator's form, on the device (pp_events_decode_kernel).
int serfsim_wire_decode_events_batch(serfsim_t* h, const uint8_t* buf, const uint64_t* offsets, uint32_t n, uint64_t* event_ltime, uint32_t* seen, uint32_t* n_unmatched) {
  if (!h || !buf || !offsets || !event_ltime || !seen || !n_unmatched) return serfsim_fail(SERFSIM_E_INVAL, "null argument");
  WireView v{};
  int rc = serfsim_wire_view(h, &v);
  if (rc) return rc;
  if (!v.ue.n) return serfsim_fail(SERFSIM_E_INVAL, "wire: no user-event content table (serfsim_set_user_event_content)");
  if ((rc = check_batch_offsets(offsets, n))) return rc;
  if (!n) return 0;                                          // nothing to decode
  const size_t total = (size_t)offsets[n];
  DevArray<u8> d_buf;
  DevArray<u64> d_off, d_ev;
  DevArray<u32> d_seen, d_um, d_err;
  CU(d_buf.alloc(total ? total : 1)); CU(d_off.alloc((size_t)n + 1)); CU(d_ev.alloc(n));
  CU(d_seen.alloc(n)); CU(d_um.alloc(n)); CU(d_err.alloc(n));
  CU(cudaMemcpyAsync(d_buf, buf, total, cudaMemcpyHostToDevice, v.stream));
  CU(cudaMemcpyAsync(d_off, offsets, d_off.bytes(), cudaMemcpyHostToDevice, v.stream));
  SFS_LAUNCH((n + 127) / 128, 128, 0, v.stream, pp_events_decode_kernel)(d_buf.get(), d_off.get(), n, v.ue, d_ev.get(), d_seen.get(), d_um.get(), d_err.get());
  std::vector<u32> err(n);
  CU(cudaMemcpyAsync(event_ltime, d_ev, d_ev.bytes(), cudaMemcpyDeviceToHost, v.stream));
  CU(cudaMemcpyAsync(seen, d_seen, d_seen.bytes(), cudaMemcpyDeviceToHost, v.stream));
  CU(cudaMemcpyAsync(n_unmatched, d_um, d_um.bytes(), cudaMemcpyDeviceToHost, v.stream));
  CU(cudaMemcpyAsync(err.data(), d_err, d_err.bytes(), cudaMemcpyDeviceToHost, v.stream));
  CU(cudaStreamSynchronize(v.stream));
  CU(cudaGetLastError());
  for (u32 i = 0; i < n; ++i)
    if (err[i] & 0x80000000u) { werr(-(int)(err[i] & 0xffffu)); return serfsim_fail(SERFSIM_E_INVAL, (std::string("wire: message ") + std::to_string(i) + ": " + serfsim_last_error()).c_str()); }
  return 0;
}

}  // extern "C"
#pragma GCC visibility pop
