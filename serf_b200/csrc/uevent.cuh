// uevent.cuh — user-event dissemination rules (SURVEY §8f row 3), shared by the device kernel and the host-compiled
// rule check in tests/cpp/uevent_rules_check.cpp (everything here is __host__ __device__ and free of memory traffic).
//
// What is restated (reference paths relative to serf-core/src):
//   Serf::user_event            serf/api.rs:241-299   — ltime = event_clock.time(); event_clock.increment();
//                                                        handle_user_event(msg) (result IGNORED); queue_broadcast(raw)
//   Serf::handle_user_event     serf/base.rs:750-837  — witness; `ltime < min_time` → drop; "too old" window of
//                                                        event_buffer_size (512, options.rs:517); ring slot ltime % 512;
//                                                        occupied slot: equal (name, payload) → drop, else push — the slot's
//                                                        own ltime is neither checked nor refreshed (SURVEY §8c quirk ii);
//                                                        returns true → SerfDelegate::notify_message re-queues the raw bytes
//                                                        (serf/delegate.rs:219-221, 293-300) with a fresh transmit budget
//   event queue drain           serf/delegate.rs:317-384 — event broadcasts ride in the same gossip packets as intents
//
// Simulation model: E ≤ 8 TRACKED user events.  Tracked event e has a host-given content id (two events with the same
// id have equal name and payload) and a Lamport time stamped by its origin when it is injected.  A node's whole event
// state is 16 bytes: event clock, `seen` mask (ring slots it filled, by tracked event), `first` mask (the lowest-index seen
// event of each occupied ring slot — derived, see ue_first_mask), and one transmit budget per event.
// Gossip entries are single bits OR-ed into the destination's inbox word: an event message carries nothing a receiver
// does not already know from the table (ltime, content), so "which tracked events arrived" is the complete payload and
// OR is the order-independent reduction (receiving k copies equals receiving one: copies 2..k are duplicates).
// Canonical order inside a tick: arrived events by ascending index, then the node's own injection.
#pragma once
#include "record.cuh"

namespace sfs {

constexpr u32 MAX_UEVENTS = 8;
constexpr u32 UE_RING = 512;                 // Options::event_buffer_size, options.rs:517
constexpr u32 OP_USER_EVENT = 6;
constexpr u32 UE_INIT_CLOCK = 1;             // Serf::new increments event_clock once (serf/base.rs:198-200; KAT serf_stats: event_time 1)

struct UeRec {                               // unpacked 16-byte event record of one node
  u32 clock;                                 // event_clock.time()
  u32 seen, first;                           // bit e: tracked event e sits in this node's ring / created its ring slot
  u32 tx[MAX_UEVENTS];                       // remaining transmits of the queued broadcast of event e
};
struct UeTable {                             // per run, by value
  u32 n;                                     // tracked events
  u32 content[MAX_UEVENTS];                  // identity of (name, payload)
};
enum : int { UE_ACCEPTED = 0, UE_DUPLICATE = 1, UE_TOO_OLD = 2 };
struct UeCounts { u32 messages, edges, delivered, duplicates, too_old, pending; };

__host__ __device__ inline void ue_unpack(const uint4& w, UeRec& r) {
  r.clock = w.x; r.seen = w.y & 0xffu; r.first = (w.y >> 8) & 0xffu;
#pragma unroll
  for (u32 e = 0; e < 4; ++e) { r.tx[e] = (w.z >> (8 * e)) & 0xffu; r.tx[4 + e] = (w.w >> (8 * e)) & 0xffu; }
}
__host__ __device__ inline uint4 ue_pack(const UeRec& r) {
  uint4 w;
  w.x = r.clock; w.y = r.seen | (r.first << 8); w.z = 0; w.w = 0;
#pragma unroll
  for (u32 e = 0; e < 4; ++e) { w.z |= (r.tx[e] & 0xffu) << (8 * e); w.w |= (r.tx[4 + e] & 0xffu) << (8 * e); }
  return w;
}

// `first` is a DERIVED field: bit e is set iff e is the lowest-index seen event of its ring slot (class = ltime % 512).
// It depends only on the seen set and on the Lamport times of seen events (which are final once an event has been seen),
// not on the order in which the events arrived — push-pull replays a partner's ring in an order the packed record does
// not keep.  Cluster runs require that two tracked events that share a ring slot also share their Lamport time (checked
// by the host after every step; the slot-reuse quirk itself lives on in ue_handle and is pinned by the handler tests), so
// the slot's own ltime — what a push-pull replay carries — is the ltime of any event in it.
__host__ __device__ inline u32 ue_first_mask(u32 seen, const u32* ltime, u32 n) {
  u32 first = 0;
  for (u32 e = 0; e < n; ++e) {
    if (!((seen >> e) & 1u)) continue;
    bool lowest = true;
    for (u32 j = 0; j < e; ++j) if (((seen >> j) & 1u) && ltime[j] % UE_RING == ltime[e] % UE_RING) lowest = false;
    if (lowest) first |= 1u << e;
  }
  return first;
}

// handle_user_event (serf/base.rs:750-837) for tracked event e carried with Lamport time L (its own, or — in a push-pull
// replay — the partner's slot ltime); `ltime[j]` is read only for events in `seen` and for e itself.  `self_L`: the event
// is being stamped by this very call (the table entry is not written yet).
__host__ __device__ inline int ue_handle(UeRec& r, u32 e, u32 L, const u32* ltime, const UeTable& tb, u32 limit, bool requeue, bool self_L = false) {
  witness(r.clock, L);                                                   // :763
  // :766-768 `ltime < min_time`: min_time stays 0 here (it only moves on a join with event_join_ignore, delegate.rs:531-537)
  if (r.clock > UE_RING && L < r.clock - UE_RING) return UE_TOO_OLD;     // :771-781
  const u32 idx = L % UE_RING;                                           // :784
  for (u32 j = 0; j < tb.n; ++j) {
    if (!((r.seen >> j) & 1u)) continue;
    if (ltime[j] % UE_RING != idx) continue;                             // the slot exists, whatever ltime it was created with (quirk ii)
    if (tb.content[j] == tb.content[e]) return UE_DUPLICATE;             // :801-806
  }
  r.seen |= 1u << e;                                                     // :807 push, or :809-813 new slot
  {                                                                      // re-derive `first` (see ue_first_mask); e's own time may not be in the table yet
    u32 lt[MAX_UEVENTS];
    for (u32 j = 0; j < tb.n; ++j) lt[j] = (j == e && self_L) ? L : ltime[j];
    r.first = ue_first_mask(r.seen, lt, tb.n);
  }
  if (requeue) r.tx[e] = limit;                                          // → true → re-queued, delegate.rs:293-300
  return UE_ACCEPTED;
}

// Serf::user_event (serf/api.rs:241-299) at the origin; returns the stamped Lamport time.
__host__ __device__ inline u32 ue_originate(UeRec& r, u32 e, const u32* ltime, const UeTable& tb, u32 limit, int& outcome) {
  const u32 L = r.clock;                                                 // :264
  r.clock += 1;                                                          // :285 increment
  outcome = ue_handle(r, e, L, ltime, tb, limit, false, true);           // :288, result ignored
  r.tx[e] = limit;                                                       // :290-297 queued unconditionally
  return L;
}

// Push-pull replay (SerfDelegate::merge_remote_state, serf/delegate.rs:466-468 and 539-552): witness the partner's event
// clock − 1, then hand every event of the partner's ring to handle_user_event with the slot's ltime — nothing is re-queued.
// Replay order: ring index ascending, as the reference walks its buffer (it matters: every replay witnesses its ltime,
// and a later event can thereby fall out of the 512-wide window); inside a slot the packed record keeps no order and none
// is needed (one ltime per slot in cluster runs, acceptance per content, `first` derived) — ascending event index.
__host__ __device__ inline void ue_replay(UeRec& r, u32 partner_clock, u32 partner_seen, const u32* ltime, const UeTable& tb, u32 limit, UeCounts& c) {
  if (partner_clock > 0) witness(r.clock, partner_clock - 1);
  u32 todo = partner_seen & ((1u << tb.n) - 1u);
  while (todo) {
    u32 best = 0, best_key = 0xffffffffu;
    for (u32 e = 0; e < tb.n; ++e) {
      if (!((todo >> e) & 1u)) continue;
      const u32 key = ((ltime[e] % UE_RING) << 4) | e;
      if (key < best_key) { best_key = key; best = e; }
    }
    todo &= ~(1u << best);
    const int oc = ue_handle(r, best, ltime[best], ltime, tb, limit, false);
    if (oc == UE_ACCEPTED) c.delivered++; else if (oc == UE_DUPLICATE) c.duplicates++; else c.too_old++;
  }
}

// Gossip send of one node to its `nt` targets (target k gets event e iff its remaining budget exceeds k — one
// get_broadcasts call per target, each counting one transmit): fills bits[k], decrements the budgets.
template <int FMAX>
__host__ __device__ inline u32 ue_plan_send(UeRec& r, u32 n_events, u32 nt, u32 (&bits)[FMAX]) {
  u32 msgs = 0;
#pragma unroll
  for (int k = 0; k < FMAX; ++k) bits[k] = 0;
  for (u32 e = 0; e < n_events; ++e) {
    const u32 tx = r.tx[e];
    if (!tx) continue;
#pragma unroll
    for (int k = 0; k < FMAX; ++k)
      if ((u32)k < nt && tx > (u32)k) { bits[k] |= 1u << e; ++msgs; }
    r.tx[e] = tx - (tx < nt ? tx : nt);
  }
  return msgs;
}
__host__ __device__ inline u32 ue_queued(const UeRec& r, u32 n_events) {
  u32 q = 0;
  for (u32 e = 0; e < n_events; ++e) q += r.tx[e] ? 1u : 0u;
  return q;
}
__host__ __device__ inline u64 ue_hash(u64 idx, const uint4& w) {
  return mix64((((u64)w.y << 32) | w.x) ^ mix64((((u64)w.w << 32) | w.z) ^ mix64(idx + 0x9e3779b97f4a7c15ULL)));
}


// Gossip peers of node v at tick t: the draw every sender makes (record.cuh peer_issue), user events ride in the same packets.
__host__ __device__ inline u32 ue_pick_targets(u32 tick, u32 v, u32 row0, u32 deg, u32 fanout, u32 seed_lo, u32 seed_hi, const u32* col, u32 (&tg)[MAX_FANOUT]) {
  u32 cand[MAX_FANOUT];
  peer_issue<(int)MAX_FANOUT>(tick, v, fanout, seed_lo, seed_hi, row0, deg, [&](u32 e) { return col[e]; }, cand);
  return peer_finish<(int)MAX_FANOUT>(v, cand, tg);
}

// Phases R and E of one node (pure): arrived events by ascending index, then the node's own injection.
// Returns the Lamport time stamped by an injection (valid when op == OP_USER_EVENT and the node is up).
__host__ __device__ inline u32 ue_receive_and_originate(UeRec& r, u32 arrived, bool up_r, u32 op, u32 op_event, const u32* ltime, const UeTable& tb, u32 limit, UeCounts& c, bool& stamped) {
  stamped = false;
  u32 L = 0;
  if (up_r) {
    for (u32 e = 0; e < tb.n; ++e) {
      if (!((arrived >> e) & 1u)) continue;
      const int oc = ue_handle(r, e, ltime[e], ltime, tb, limit, true);
      if (oc == UE_ACCEPTED) c.delivered++; else if (oc == UE_DUPLICATE) c.duplicates++; else c.too_old++;
    }
    if (op == OP_USER_EVENT && op_event < tb.n) {
      int oc;
      L = ue_originate(r, op_event, ltime, tb, limit, oc);
      stamped = true;
      if (oc == UE_ACCEPTED) c.delivered++; else if (oc == UE_DUPLICATE) c.duplicates++; else c.too_old++;
    }
  }
  return L;
}

}  // namespace sfs
