// wire.cuh — serf's wire format for the messages of the hot path (SURVEY §8f row 4): Join, Leave, PushPull.
//
// Restated from serf-core/src/types/{message.rs:17-47, 397-428, 507-692; join.rs:8-158; leave.rs:8-195; push_pull.rs:100-114,
// 319-450; clock.rs:96-119}: a protobuf-like TLV stream — every field is one tag byte merge(wire type, tag) followed by its
// value; a message travels as [message byte][varint payload length][payload] (encode_message, message.rs:397-428).
//
// EXTERNAL, NOT UNDER /root/reference (memberlist_core::proto of memberlist-core 0.8.1, Cargo.toml:39-41): the helpers the
// reference calls — `merge`, `skip`, `WireType`, the varint codec of u64 / u32, `encode_length_delimited`, `TupleEncoder`.
// Their byte layout is restated here from the protobuf conventions that crate follows and is therefore UNPINNED at byte level:
//   * merge(wire, tag) = tag << 3 | wire (message tags reach 10 — message.rs:17-28 — so the tag cannot live in 3 low bits);
//   * WireType: Byte = 0, Varint = 1, LengthDelimited = 2, Fixed32 = 3, Fixed64 = 4 (only the first three occur on this path);
//   * u64 / u32 / LamportTime: LEB128 varint (7 bits per byte, least significant group first), wire type Varint;
//   * bool: one byte (wire type Byte); a u64 id: Varint, and encode_length_delimited of a non-LengthDelimited type adds no
//     length prefix; TupleEncoder(k, v) = [merge(K wire, 1)][k][merge(V wire, 2)][v] (a protobuf map entry);
//   * a `&str` / `Bytes` value and a nested message (UserEvent inside UserEvents, UserEvents inside PushPull) are
//     length-delimited as [varint byte length][bytes]; a name's UTF-8 is neither produced nor checked here (the bytes travel
//     as given).
// User events (types/user_event.rs, user_event/{user_events.rs, message.rs}; PushPullMessageBorrow, push_pull.rs:455-587) are
// restated below the PushPull part.
// Everything IN the reference tree — which fields exist, their tags, order, optionality, duplicate / missing-field errors,
// skipping of unknown fields — is followed line by line.  All layout assumptions sit in the constants below.
#pragma once
#include <cstddef>
#include <cstdint>

#ifndef __CUDACC__
#ifndef __host__
#define __host__
#define __device__
#endif
#endif

namespace sfs {
namespace wire {

typedef uint8_t u8;
typedef uint32_t u32;
typedef uint64_t u64;

enum : u8 { WT_BYTE = 0, WT_VARINT = 1, WT_LEN = 2, WT_FIXED32 = 3, WT_FIXED64 = 4 };
__host__ __device__ constexpr u8 merge(u8 wire, u8 tag) { return (u8)((tag << 3) | wire); }
__host__ __device__ constexpr u8 wire_of(u8 b) { return (u8)(b & 7u); }

// message bytes — types/message.rs:17-47
constexpr u8 MSG_LEAVE = merge(WT_LEN, 1), MSG_JOIN = merge(WT_LEN, 2), MSG_PUSH_PULL = merge(WT_LEN, 3), MSG_USER_EVENT = merge(WT_LEN, 4);
// JoinMessage — types/join.rs:8-10: ltime = 1 (varint), id = 2
constexpr u8 JOIN_LTIME = merge(WT_VARINT, 1), JOIN_ID = merge(WT_VARINT, 2);
// LeaveMessage — types/leave.rs:8-13: ltime = 1 (varint), prune = 2 (byte, written only when true, :149-156), id = 3
constexpr u8 LEAVE_LTIME = merge(WT_VARINT, 1), LEAVE_PRUNE = merge(WT_BYTE, 2), LEAVE_ID = merge(WT_VARINT, 3);
// PushPullMessage — types/push_pull.rs:100-114: ltime = 1, status_ltimes = 2 (repeated tuple), left_members = 3 (repeated id),
// event_ltime = 4, events = 5 (repeated UserEvents), query_ltime = 6
constexpr u8 PP_LTIME = merge(WT_VARINT, 1), PP_STATUS = merge(WT_LEN, 2), PP_LEFT = merge(WT_VARINT, 3), PP_EVENT_LTIME = merge(WT_VARINT, 4),
             PP_EVENTS = merge(WT_LEN, 5), PP_QUERY_LTIME = merge(WT_VARINT, 6);
constexpr u8 TUPLE_KEY = merge(WT_VARINT, 1), TUPLE_VALUE = merge(WT_VARINT, 2);
// UserEvent — types/user_event.rs:15-19: name = 1, payload = 2 (LengthDelimited; each written only when non-empty, :109-148)
constexpr u8 UE_NAME = merge(WT_LEN, 1), UE_PAYLOAD = merge(WT_LEN, 2);
// UserEvents — user_event/user_events.rs: ltime = 1 (varint, required), events = 2 (repeated LengthDelimited UserEvent)
constexpr u8 UES_LTIME = merge(WT_VARINT, 1), UES_EVENT = merge(WT_LEN, 2);
// UserEventMessage — user_event/message.rs:68-76: ltime = 1 (varint, required), cc = 2 (byte), name = 3, payload = 4
constexpr u8 UEM_LTIME = merge(WT_VARINT, 1), UEM_CC = merge(WT_BYTE, 2), UEM_NAME = merge(WT_LEN, 3), UEM_PAYLOAD = merge(WT_LEN, 4);
constexpr u32 MAX_USER_EVENT_SIZE = 512;      // Options::max_user_event_size (options.rs:528): name + payload, and the encoded message

enum : int { OK = 0, E_TRUNCATED = -1, E_VARINT = -2, E_DUPLICATE = -3, E_MISSING = -4, E_WIRE_TYPE = -5, E_CAPACITY = -6, E_TYPE = -7 };

__host__ __device__ inline u32 varint_len(u64 v) { u32 n = 1; while (v >= 0x80) { v >>= 7; ++n; } return n; }
__host__ __device__ inline u32 varint_put(u8* p, u64 v) { u32 n = 0; while (v >= 0x80) { p[n++] = (u8)(v | 0x80); v >>= 7; } p[n++] = (u8)v; return n; }
// returns bytes read (> 0) or an error (< 0)
__host__ __device__ inline int varint_get(const u8* p, size_t len, u64* out) {
  u64 v = 0;
  for (u32 i = 0; i < 10; ++i) {
    if (i >= len) return E_TRUNCATED;
    const u8 b = p[i];
    if (i == 9 && b > 1) return E_VARINT;                     // more than 64 bits
    v |= (u64)(b & 0x7f) << (7 * i);
    if (!(b & 0x80)) { *out = v; return (int)i + 1; }
  }
  return E_VARINT;
}
// memberlist_core::proto::utils::skip: the unknown field starting at its tag byte; returns bytes to skip or an error
__host__ __device__ inline long skip_field(const u8* p, size_t len) {
  if (len < 1) return E_TRUNCATED;
  u64 v;
  switch (wire_of(p[0])) {
    case WT_BYTE: return len >= 2 ? 2 : E_TRUNCATED;
    case WT_VARINT: { const int n = varint_get(p + 1, len - 1, &v); return n < 0 ? n : 1 + n; }
    case WT_LEN: { const int n = varint_get(p + 1, len - 1, &v); if (n < 0) return n; return (u64)(len - 1 - n) >= v ? (long)(1 + n + v) : (long)E_TRUNCATED; }
    case WT_FIXED32: return len >= 5 ? 5 : E_TRUNCATED;
    case WT_FIXED64: return len >= 9 ? 9 : E_TRUNCATED;
    default: return E_WIRE_TYPE;
  }
}

// ---- Join / Leave (payload = the message body; envelope = message byte + varint(payload length) + payload) ----
__host__ __device__ inline u32 join_payload_len(u64 ltime, u64 id) { return 1 + varint_len(ltime) + 1 + varint_len(id); }                       // join.rs:127-129
__host__ __device__ inline u32 leave_payload_len(u64 ltime, u64 id, bool prune) { return 1 + varint_len(ltime) + (prune ? 2u : 0u) + 1 + varint_len(id); }   // leave.rs:134-139
__host__ __device__ inline u32 envelope_len(u32 payload) { return 1 + varint_len(payload) + payload; }                                            // encoded_message_len, message.rs:484-491
__host__ __device__ inline u32 put_join(u8* p, u64 ltime, u64 id) {                   // join.rs:131-158, inside message.rs:397-428
  u32 o = 0;
  const u32 pl = join_payload_len(ltime, id);
  p[o++] = MSG_JOIN; o += varint_put(p + o, pl);
  p[o++] = JOIN_LTIME; o += varint_put(p + o, ltime);
  p[o++] = JOIN_ID; o += varint_put(p + o, id);
  return o;
}
__host__ __device__ inline u32 put_leave(u8* p, u64 ltime, u64 id, bool prune) {      // leave.rs:141-195
  u32 o = 0;
  const u32 pl = leave_payload_len(ltime, id, prune);
  p[o++] = MSG_LEAVE; o += varint_put(p + o, pl);
  p[o++] = LEAVE_LTIME; o += varint_put(p + o, ltime);
  if (prune) { p[o++] = LEAVE_PRUNE; p[o++] = 1; }
  p[o++] = LEAVE_ID; o += varint_put(p + o, id);
  return o;
}

// The envelope: decode_message (message.rs:507-692) walks the buffer, takes the first known message byte (a second one is a
// duplicate-field error) and skips unknown fields.  Returns the payload range of the single message.
__host__ __device__ inline int open_envelope(const u8* p, size_t len, u8* type, size_t* pay_off, size_t* pay_len) {
  size_t o = 0;
  bool have = false;
  while (o < len) {
    const u8 b = p[o];
    if (b == MSG_LEAVE || b == MSG_JOIN || b == MSG_PUSH_PULL || b == MSG_USER_EVENT) {
      if (have) return E_DUPLICATE;
      u64 n;
      const int r = varint_get(p + o + 1, len - o - 1, &n);
      if (r < 0) return r;
      if ((u64)(len - o - 1 - r) < n) return E_TRUNCATED;
      *type = b; *pay_off = o + 1 + r; *pay_len = (size_t)n; have = true;
      o += 1 + r + (size_t)n;
    } else {
      const long s = skip_field(p + o, len - o);
      if (s < 0) return (int)s;
      o += (size_t)s;
    }
  }
  return have ? OK : E_MISSING;
}
struct Intent { u64 ltime, id; bool prune; };
// JoinMessage::decode (join.rs:54-111) / LeaveMessage::decode (leave.rs:56-119) on the payload
__host__ __device__ inline int get_intent(const u8* p, size_t len, bool leave, Intent* out) {
  size_t o = 0;
  bool has_lt = false, has_id = false, has_prune = false;
  out->prune = false;
  while (o < len) {
    const u8 b = p[o];
    if (b == (leave ? LEAVE_LTIME : JOIN_LTIME)) {
      if (has_lt) return E_DUPLICATE;
      const int r = varint_get(p + o + 1, len - o - 1, &out->ltime);
      if (r < 0) return r;
      o += 1 + r; has_lt = true;
    } else if (leave && b == LEAVE_PRUNE) {
      if (has_prune) return E_DUPLICATE;
      if (len - o < 2) return E_TRUNCATED;
      out->prune = p[o + 1] != 0; o += 2; has_prune = true;
    } else if (b == (leave ? LEAVE_ID : JOIN_ID)) {
      if (!leave && has_id) return E_DUPLICATE;               // join.rs:80-82 rejects a second id; leave.rs:103-108 keeps the last one
      const int r = varint_get(p + o + 1, len - o - 1, &out->id);
      if (r < 0) return r;
      o += 1 + r; has_id = true;
    } else {
      const long s = skip_field(p + o, len - o);
      if (s < 0) return (int)s;
      o += (size_t)s;
    }
  }
  return (has_lt && has_id) ? OK : E_MISSING;
}

// ---- PushPull ----
__host__ __device__ inline u32 tuple_len(u64 id, u64 st) { return 1 + varint_len(id) + 1 + varint_len(st); }
__host__ __device__ inline u32 pp_status_entry_len(u64 id, u64 st) { const u32 t = tuple_len(id, st); return 1 + varint_len(t) + t; }   // push_pull.rs:349-353
__host__ __device__ inline u32 pp_left_entry_len(u64 id) { return 1 + varint_len(id); }                                             // :355-359
__host__ __device__ inline u32 put_pp_status_entry(u8* p, u64 id, u64 st) {                                                         // :388-398
  u32 o = 0;
  p[o++] = PP_STATUS; o += varint_put(p + o, tuple_len(id, st));
  p[o++] = TUPLE_KEY; o += varint_put(p + o, id);
  p[o++] = TUPLE_VALUE; o += varint_put(p + o, st);
  return o;
}

// ---- user events ----
// A length-delimited value after its tag byte: [varint n][n bytes].  Returns the bytes taken (> 0) or an error; *off / *n give
// the value's range relative to p.
__host__ __device__ inline int get_len_delim(const u8* p, size_t len, u32* off, u32* n) {
  u64 v;
  const int r = varint_get(p, len, &v);
  if (r < 0) return r;
  if ((u64)(len - r) < v) return E_TRUNCATED;
  *off = (u32)r; *n = (u32)v;
  return r + (int)v;
}
__host__ __device__ inline u32 len_delim_len(u32 n) { return 1 + varint_len(n) + n; }        // tag + length + bytes
__host__ __device__ inline u32 put_len_delim(u8* p, u8 tag, const u8* v, u32 n) {
  u32 o = 0;
  p[o++] = tag; o += varint_put(p + o, n);
  for (u32 i = 0; i < n; ++i) p[o + i] = v[i];
  return o + n;
}
// UserEvent body (user_event.rs:109-148): name, then payload, each only when non-empty
__host__ __device__ inline u32 user_event_len(u32 nl, u32 pl) { return (nl ? len_delim_len(nl) : 0u) + (pl ? len_delim_len(pl) : 0u); }
__host__ __device__ inline u32 put_user_event(u8* p, const u8* name, u32 nl, const u8* pay, u32 pl) {
  u32 o = 0;
  if (nl) o += put_len_delim(p + o, UE_NAME, name, nl);
  if (pl) o += put_len_delim(p + o, UE_PAYLOAD, pay, pl);
  return o;
}
// One entry of UserEvents.events (user_events.rs encode: [events byte][UserEvent, length-delimited]) — the unit the batch
// encoder copies from the content table.
__host__ __device__ inline u32 ues_event_entry_len(u32 nl, u32 pl) { return len_delim_len(user_event_len(nl, pl)); }
// One PushPull `events` entry (push_pull.rs:566-577): [events byte][UserEvents{ltime, events}, length-delimited], the events
// entries summing to `entries` bytes.
__host__ __device__ inline u32 ues_body_len(u64 ltime, u64 entries) { return 1 + varint_len(ltime) + (u32)entries; }
__host__ __device__ inline u32 pp_events_entry_len(u64 ltime, u64 entries) { return len_delim_len(ues_body_len(ltime, entries)); }
__host__ __device__ inline u32 put_pp_events_head(u8* p, u64 ltime, u64 entries) {        // everything of the entry before its events
  u32 o = 0;
  p[o++] = PP_EVENTS; o += varint_put(p + o, ues_body_len(ltime, entries));
  p[o++] = UES_LTIME; o += varint_put(p + o, ltime);
  return o;
}

// UserEventMessage (user_event/message.rs:206-271): ltime, cc only when true, name if non-empty, payload if non-empty
__host__ __device__ inline u32 uem_payload_len(u64 ltime, u32 nl, u32 pl, bool cc) {
  return 1 + varint_len(ltime) + (cc ? 2u : 0u) + user_event_len(nl, pl);
}
__host__ __device__ inline u32 put_uem(u8* p, u64 ltime, const u8* name, u32 nl, const u8* pay, u32 pl, bool cc) {   // with the envelope
  u32 o = 0;
  p[o++] = MSG_USER_EVENT; o += varint_put(p + o, uem_payload_len(ltime, nl, pl, cc));
  p[o++] = UEM_LTIME; o += varint_put(p + o, ltime);
  if (cc) { p[o++] = UEM_CC; p[o++] = 1; }
  if (nl) o += put_len_delim(p + o, UEM_NAME, name, nl);
  if (pl) o += put_len_delim(p + o, UEM_PAYLOAD, pay, pl);
  return o;
}

// Decoded byte ranges are offsets into the decoded buffer (no copy).
struct EventBytes { u32 name_off, name_len, pay_off, pay_len; };
// UserEventRef::decode (user_event.rs:51-95) on a body at p[0, len); offsets are relative to `base`.  Both fields default to
// empty; a second name or payload is a duplicate-field error; unknown fields are skipped.
__host__ __device__ inline int get_user_event(const u8* p, size_t len, u32 base, u8 name_tag, u8 pay_tag, EventBytes* out, bool* cc = nullptr, u64* ltime = nullptr) {
  size_t o = 0;
  bool hn = false, hp = false, hc = false, hl = false;
  *out = EventBytes{0, 0, 0, 0};
  while (o < len) {
    const u8 b = p[o];
    if (b == name_tag || b == pay_tag) {
      bool& have = b == name_tag ? hn : hp;
      if (have) return E_DUPLICATE;
      u32 off, n;
      const int r = get_len_delim(p + o + 1, len - o - 1, &off, &n);
      if (r < 0) return r;
      if (b == name_tag) { out->name_off = base + (u32)(o + 1) + off; out->name_len = n; }
      else { out->pay_off = base + (u32)(o + 1) + off; out->pay_len = n; }
      have = true; o += 1 + r;
    } else if (ltime && b == UEM_LTIME) {                   // UserEventMessage only (message.rs:103-117)
      if (hl) return E_DUPLICATE;
      const int r = varint_get(p + o + 1, len - o - 1, ltime);
      if (r < 0) return r;
      hl = true; o += 1 + r;
    } else if (cc && b == UEM_CC) {                         // :118-131
      if (hc) return E_DUPLICATE;
      if (len - o < 2) return E_TRUNCATED;
      *cc = p[o + 1] != 0; hc = true; o += 2;
    } else {
      const long s = skip_field(p + o, len - o);
      if (s < 0) return (int)s;
      o += (size_t)s;
    }
  }
  if (cc && !hc) *cc = false;
  return (ltime && !hl) ? E_MISSING : OK;                   // :181 ltime is required; the rest defaults
}
__host__ __device__ inline int get_uem(const u8* p, size_t len, u32 base, u64* ltime, EventBytes* ev, bool* cc) {
  return get_user_event(p, len, base, UEM_NAME, UEM_PAYLOAD, ev, cc, ltime);
}

// UserEventsRef::decode + UserEvents::from_ref (user_events.rs): the body of one PushPull `events` entry at p[0, len), offsets
// relative to `base`.  ltime is required and single; every events field is decoded as a UserEvent (an error in one fails the
// entry); unknown fields are skipped.  on_event(const EventBytes&) is called per event, in order, after the whole entry has
// been validated (ltime may come after the events); it returns OK or an error that ends the walk.
template <class F>
__host__ __device__ inline int walk_user_events(const u8* p, size_t len, u32 base, u64* ltime, u32* n_events, F&& on_event) {
  bool hl = false;
  u32 ne = 0;
  for (int pass = 0; pass < 2; ++pass) {
    size_t o = 0;
    while (o < len) {
      const u8 b = p[o];
      if (b == UES_LTIME && pass == 0) {
        if (hl) return E_DUPLICATE;
        const int r = varint_get(p + o + 1, len - o - 1, ltime);
        if (r < 0) return r;
        hl = true; o += 1 + r;
      } else if (b == UES_EVENT) {
        u32 off, n;
        const int r = get_len_delim(p + o + 1, len - o - 1, &off, &n);
        if (r < 0) return r;
        const u32 at = (u32)(o + 1) + off;
        EventBytes ev;
        const int rc = get_user_event(p + at, n, base + at, UE_NAME, UE_PAYLOAD, &ev);
        if (rc) return rc;
        if (pass == 0) ++ne;
        else { const int rc2 = on_event(ev); if (rc2) return rc2; }
        o += 1 + r;
      } else {
        const long s = skip_field(p + o, len - o);
        if (s < 0) return (int)s;
        o += (size_t)s;
      }
    }
    if (pass == 0 && !hl) return E_MISSING;
  }
  *n_events = ne;
  return OK;
}

// The wire form of the tracked user events as the batch kernels see it (serfsim_set_user_event_content): entry e of
// `entries` is the UserEvents.events entry of tracked event e; its name / payload ranges are kept for decode-side matching.
constexpr u32 UE_TABLE_MAX = 8;                                            // = SERFSIM_MAX_USER_EVENTS
constexpr u32 UE_ENTRY_MAX = 1 + 2 + 2 * (1 + 2) + MAX_USER_EVENT_SIZE;    // one entry: tag, 2-byte lengths, ≤ 512 content bytes
struct UeWire {
  u32 n;                                  // tracked events with content; 0 = no content table (no events are attached)
  const u8* entries;                      // device: the n entries back to back
  const u32* ltime;                       // device: the Lamport time of each tracked event (0: not fired)
  u32 off[UE_TABLE_MAX + 1];              // entry e = entries[off[e], off[e + 1])
  EventBytes bytes[UE_TABLE_MAX];         // name / payload of e, relative to entries
};

}  // namespace wire
}  // namespace sfs
