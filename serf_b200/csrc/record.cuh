// record.cuh — the 32-byte member record and the per-record transition rules (device side).
//
// One record = one node's view of one tracked subject.  The rules are the reference's
// (serf-core/src/serf/base.rs, types/clock.rs) restated for a batch: the inbox of a
// (node, slot) holds only the REDUCED message set of the tick — the greatest leave-intent
// Lamport time, the greatest join-intent Lamport time, the greatest memberlist key — and
// applying those three in the order memberlist → leave → join gives exactly the state that
// applying every received message one at a time (leaves ascending, then joins ascending)
// would: status transitions are idempotent, status_time only moves up, and a lower message
// of a kind is accepted only if the greatest one is (DESIGN.md "Reduction lemma").
//
// Layout (little endian, 32 B = one DRAM sector):
//    0 u32 status_ltime   MemberState.status_time (types/member.rs:23); buffered-intent ltime while !known
//    4 u32 qjoin_lt       Lamport time of the queued join intent   (SerfBroadcast, broadcast.rs:15-45)
//    8 u32 qleave_lt      Lamport time of the queued leave intent
//   12 u32 incarnation    memberlist incarnation of the subject as seen by this node
//   16 u32 deadline       tick at which the suspicion timer fires, 0 = none
//   20 u32 leave_tick     MemberState.leave_time as tick+1, 0 = None (types/member.rs:25)
//   24 u8  status         MemberStatus (types/member.rs:54-58); buffered-intent MessageType while !known
//   25 u8  ml             bits 0-1 memberlist state, bits 2-5 from-bucket of the queued suspect
//   26 u8  tx_join        remaining transmits of the queued join intent (TransmitLimitedQueue)
//   27 u8  tx_leave       remaining transmits of the queued leave intent
//   28 u8  tx_ml          remaining transmits of the queued alive/suspect/dead message
//   29 u8  flags          bit 0: known (member present in Members.states, types/member.rs:37); bit 1: the queued leave intent carries
//                         LeaveMessage.prune (types/leave.rs:39-44)
//   30 u16 conf_mask      suspicion confirmer buckets (Lifeguard)
#pragma once
#include <cstddef>
#include <cstdint>

// Small format and rule helpers are force-inlined under nvcc, as the kernel code they serve: the tick kernels' machine code
// depends on the point at which a helper is inlined.
#ifdef __CUDACC__
#define SFS_HD __host__ __device__ __forceinline__
#else
#define SFS_HD inline
#endif

namespace sfs {

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

enum : u32 { ST_NONE = 0, ST_ALIVE = 1, ST_LEAVING = 2, ST_LEFT = 3, ST_FAILED = 4 };   // types/member.rs:54-58
enum : u32 { TY_NONE = 0, TY_LEAVE = 1, TY_JOIN = 2 };                                   // types/message.rs:17-18
enum : u32 { ML_ALIVE = 0, ML_SUSPECT = 1, ML_DEAD = 2, ML_LEFT = 3 };
enum : u32 { SS_ALIVE = 0, SS_LEAVING = 1, SS_LEFT = 2 };                                // SerfState
enum : u32 { OP_JOIN = 1, OP_LEAVE = 2, OP_FORCE_LEAVE = 3, OP_FAIL = 4, OP_REJOIN = 5, /* 6: OP_USER_EVENT, uevent.cuh */ OP_FORCE_LEAVE_PRUNE = 7 };
enum : u32 { DOMAIN_GOSSIP = 0, DOMAIN_PROBE = 1, DOMAIN_PUSHPULL = 2 };
enum : u32 { KIND_LEAVE = 0, KIND_JOIN = 1, KIND_ML = 2 };

constexpr u32 MAX_SLOTS = 16;
constexpr u32 MAX_FANOUT = 8;
constexpr u32 MAX_K = 7;            // suspicion_mult - 2
constexpr u32 LTIME_LIMIT = 0x7FFFFFF0u;     // a leave intent travels as (ltime << 1 | !prune) + 1 in 32 bits
constexpr u32 FLAG_KNOWN = 1u, FLAG_QPRUNE = 2u;
constexpr u32 INC_LIMIT = (1u << 26) - 16;

// node_state word: bits 0-31 LamportClock (types/clock.rs:125), 32 up, 40-41 SerfState
constexpr u64 NS_UP = 1ull << 32;
SFS_HD u64 node_word(u32 clock, bool up, u32 sstate) { return (u64)clock | (up ? NS_UP : 0) | ((u64)sstate << 40); }
SFS_HD u32 nw_clock(u64 ns) { return (u32)ns; }
SFS_HD bool nw_up(u64 ns) { return (ns & NS_UP) != 0; }
SFS_HD u32 nw_sstate(u64 ns) { return (u32)(ns >> 40) & 3; }

// busy byte of a node: bit 0 awake (queued transmits / probe duty), bit 1 host operation this tick, bit 2 watcher (static),
// bit 3 some view of the node runs a suspicion timer (it sleeps until its tile comes due, tick_kernel.cuh)
constexpr u32 BUSY_AWAKE = 1u, BUSY_OP = 2u, BUSY_WATCH = 4u, BUSY_TIMER = 8u;

struct Rec {
  u32 st, qjoin, qleave, inc, deadline, leave_tick;
  u32 status, mlstate, qfrom, txj, txl, txm, flags, mask;
};

// The 32-byte image of a record as eight words (layout above).  In memory a record is two uint4 (one sector).
struct Words { u32 w[8]; };
SFS_HD Words rec_words(const uint4& a, const uint4& b) { return Words{{a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w}}; }
SFS_HD Words load_rec(const uint4* rec, size_t i) { return rec_words(rec[2 * i], rec[2 * i + 1]); }
SFS_HD void store_rec(uint4* rec, size_t i, const Words& x) {
  rec[2 * i] = uint4{x.w[0], x.w[1], x.w[2], x.w[3]}; rec[2 * i + 1] = uint4{x.w[4], x.w[5], x.w[6], x.w[7]};
}
SFS_HD bool differs(const Words& a, const Words& b) {
  return ((a.w[0] ^ b.w[0]) | (a.w[1] ^ b.w[1]) | (a.w[2] ^ b.w[2]) | (a.w[3] ^ b.w[3]) | (a.w[4] ^ b.w[4]) | (a.w[5] ^ b.w[5]) | (a.w[6] ^ b.w[6]) | (a.w[7] ^ b.w[7])) != 0;
}

SFS_HD void unpack(const Words& x, Rec& r) {
  r.st = x.w[0]; r.qjoin = x.w[1]; r.qleave = x.w[2]; r.inc = x.w[3]; r.deadline = x.w[4]; r.leave_tick = x.w[5];
  r.status = x.w[6] & 0xff; r.mlstate = (x.w[6] >> 8) & 3; r.qfrom = (x.w[6] >> 10) & 15; r.txj = (x.w[6] >> 16) & 0xff; r.txl = x.w[6] >> 24;
  r.txm = x.w[7] & 0xff; r.flags = (x.w[7] >> 8) & 0xff; r.mask = x.w[7] >> 16;
}
SFS_HD void unpack(const uint4& a, const uint4& b, Rec& r) { unpack(rec_words(a, b), r); }   // a record as its two halves in memory
SFS_HD void pack(const Rec& r, Words& x) {
  x.w[0] = r.st; x.w[1] = r.qjoin; x.w[2] = r.qleave; x.w[3] = r.inc; x.w[4] = r.deadline; x.w[5] = r.leave_tick;
  x.w[6] = r.status | (r.mlstate << 8) | (r.qfrom << 10) | (r.txj << 16) | (r.txl << 24);
  x.w[7] = r.txm | (r.flags << 8) | (r.mask << 16);
}

// Queue word: the three transmit budgets of a view live in their own 4-byte plane (byte 0 tx_join, 1 tx_leave, 2 tx_ml),
// so that a sender which only decrements budgets rewrites 4 bytes instead of its whole 32-byte record.  Every external
// image of a record (records getter, state hash, oracle comparison) is the MERGED one: record | budgets.
SFS_HD void merge_queue_word(Words& x, u32 q) { x.w[6] |= ((q & 0xffu) << 16) | (((q >> 8) & 0xffu) << 24); x.w[7] |= (q >> 16) & 0xffu; }
SFS_HD u32 split_queue_word(Words& x) {
  const u32 q = ((x.w[6] >> 16) & 0xffu) | ((x.w[6] >> 24) << 8) | ((x.w[7] & 0xffu) << 16);
  x.w[6] &= 0x0000ffffu; x.w[7] &= ~0xffu;
  return q;
}
SFS_HD bool rec_queued(const Rec& r) { return (r.txl | r.txj | r.txm) != 0; }

struct Rules {          // per-run constants
  u32 limit;            // memberlist retransmit limit = retransmit_mult * ceil(log10(n+1))
  u32 k;                // max suspicion confirmations
  u32 timeout[MAX_K + 1];
};

// LamportClock::witness — types/clock.rs:155-172
__host__ __device__ inline void witness(u32& c, u32 t) { if (t >= c) c = t + 1; }

__host__ __device__ inline u32 from_bucket(u32 node) { return (node * 0x9E3779B1u) >> 28; }
SFS_HD u32 popc(u32 x) {
#ifdef __CUDA_ARCH__
  return (u32)__popc(x);
#else
  return (u32)__builtin_popcount(x);
#endif
}

// handle_node_join_intent — serf/base.rs:1338-1373 (witness by the caller); re-queue = serf/delegate.rs:294-300
__host__ __device__ inline void join_intent(Rec& r, u32 lt, u32 limit, bool requeue = true) {
  bool acc;
  if (r.flags & 1) {
    if (lt <= r.st) return;                               // :1346
    r.st = lt;                                            // :1351
    if (r.status == ST_LEAVING) r.status = ST_ALIVE;      // :1356-1358
    acc = true;
  } else {                                                // upsert_intent, :1838-1866
    acc = (r.status == TY_NONE) || (lt > r.st);
    if (acc) { r.status = TY_JOIN; r.st = lt; }
  }
  if (acc && requeue) { r.qjoin = lt; r.txj = limit; }   // push-pull discards the handler's result (serf/delegate.rs:495-523)
}

// Leave intents on the wire (inbox words, window entries): key = ltime << 1 | !prune.  Of the leave intents a view receives in
// one tick only the greatest key is applied (DESIGN.md reduction lemma); rule P-1: a prune flag carried by any other one is
// dropped — and at equal Lamport time the intent WITHOUT prune is the greater one, so that applying the greatest alone equals
// applying all of them in ascending order with the lesser ones' flags dropped.
__host__ __device__ inline u32 leave_key(u32 lt, bool prune) { return (lt << 1) | (prune ? 0u : 1u); }
SFS_HD u32 leave_key_lt(u32 key) { return key >> 1; }
SFS_HD bool leave_key_prune(u32 key) { return !(key & 1u); }

// handle_node_leave_intent — serf/base.rs:1442-1572; prune → handle_prune, :1504-1570, 1628-1653: the member is erased from the
// view (erase_node!, :499-519).  The reference sleeps broadcast_timeout + leave_propagate_delay first when the member is Leaving,
// holding the node's member lock; the tick model erases at once (as the literal oracle node does).
__host__ __device__ inline void leave_intent(Rec& r, u32 lt, bool prune, bool self, u32 sstate, bool& refute, u32 limit, bool requeue = true) {
  bool acc;
  if (!(r.flags & 1)) {                                   // :1450-1458
    acc = (r.status == TY_NONE) || (lt > r.st);
    if (acc) { r.status = TY_LEAVE; r.st = lt; }
  } else {
    if (lt <= r.st) return;                               // :1464
    if (self && sstate == SS_ALIVE) { refute = true; return; }   // :1470-1480
    r.st = lt;                                            // :1497 always
    switch (r.status) {
      case ST_NONE: acc = false; break;                   // :1501
      case ST_ALIVE: r.status = ST_LEAVING; acc = true; break;
      case ST_LEAVING: case ST_LEFT: acc = true; break;
      case ST_FAILED: r.status = ST_LEFT; acc = true; break;      // :1520-1559
      default: r.status = ST_LEAVING; acc = true; break;          // :1560-1570
    }
    if (acc && prune) { r.flags &= ~FLAG_KNOWN; r.status = TY_NONE; r.st = 0; r.leave_tick = 0; }   // handle_prune → erase_node!
  }
  if (acc && requeue) { r.qleave = lt; r.txl = limit; r.flags = (r.flags & ~FLAG_QPRUNE) | (prune ? FLAG_QPRUNE : 0u); }
}

// handle_node_join — serf/base.rs:1206-1334
__host__ __device__ inline void node_join(Rec& r) {
  if (r.flags & 1) { r.status = ST_ALIVE; r.leave_tick = 0; return; }      // :1251-1263
  u32 status = ST_ALIVE, st = 0;                                           // :1276-1288
  if (r.status == TY_JOIN) st = r.st;
  if (r.status == TY_LEAVE) { st = r.st; status = ST_LEAVING; }
  r.status = status; r.st = st; r.flags |= 1; r.leave_tick = 0;
}
// handle_node_leave — serf/base.rs:1375-1440
__host__ __device__ inline void node_leave(Rec& r, u32 tick) {
  if (!(r.flags & 1)) return;
  if (r.status == ST_LEAVING) { r.status = ST_LEFT; r.leave_tick = tick + 1; }
  else if (r.status == ST_ALIVE) { r.status = ST_FAILED; r.leave_tick = tick + 1; }
}

// memberlist (external crate memberlist-core 0.8.1; restated: aliveNode / suspectNode / deadNode / refute)
__host__ __device__ inline void ml_refute(Rec& r, u32 accused, u32 limit) {
  u32 inc = r.inc + 1;
  if (accused >= inc) inc = accused + 1;
  r.inc = inc; r.mlstate = ML_ALIVE; r.qfrom = 0; r.txm = limit;
}
__host__ __device__ inline void ml_alive(Rec& r, u32 a, bool self, u32 limit) {
  if (a <= r.inc) return;
  if (self) { ml_refute(r, a, limit); return; }
  r.deadline = 0; r.mask = 0;
  u32 old = r.mlstate;
  r.inc = a; r.mlstate = ML_ALIVE; r.qfrom = 0; r.txm = limit;
  if (old == ML_DEAD || old == ML_LEFT) node_join(r);           // EventDelegate::notify_join, serf/delegate.rs:565
}
__host__ __device__ inline void ml_suspect(Rec& r, u32 s, u32 fromb, u32 tick, bool self, const Rules& cx) {
  if (s < r.inc) return;
  if (r.mlstate == ML_SUSPECT) {                                // timer exists → suspicion.Confirm(from)
    u32 n_old = popc(r.mask) - 1;
    if (n_old >= cx.k) return;
    if (r.mask & (1u << fromb)) return;
    r.mask |= (1u << fromb);
    r.deadline = r.deadline - cx.timeout[n_old] + cx.timeout[n_old + 1];
    r.qfrom = fromb; r.txm = cx.limit;
    return;
  }
  if (r.mlstate != ML_ALIVE) return;
  if (self) { ml_refute(r, s, cx.limit); return; }
  r.inc = s; r.mlstate = ML_SUSPECT; r.qfrom = fromb; r.mask = 1u << fromb;
  r.deadline = tick + cx.timeout[0]; r.txm = cx.limit;
}
__host__ __device__ inline void ml_dead(Rec& r, u32 d, bool left, u32 tick, bool self, u32 limit) {
  if (d < r.inc) return;
  r.deadline = 0; r.mask = 0;
  if (r.mlstate == ML_DEAD || r.mlstate == ML_LEFT) return;
  if (self) { ml_refute(r, d, limit); return; }
  r.inc = d; r.mlstate = left ? ML_LEFT : ML_DEAD; r.qfrom = 0; r.txm = limit;
  node_leave(r, tick);                                          // EventDelegate::notify_leave, serf/delegate.rs:571
}
// Memberlist messages on the wire (inbox words, window entries): key = incarnation << 6 | state << 4 | from-bucket.
__host__ __device__ inline u32 ml_key(const Rec& r) { return (r.inc << 6) | (r.mlstate << 4) | r.qfrom; }
SFS_HD u32 ml_key_inc(u32 key) { return key >> 6; }
SFS_HD u32 ml_key_state(u32 key) { return (key >> 4) & 3; }
SFS_HD u32 ml_key_from(u32 key) { return key & 15; }

// Rules a view is held to after its messages were merged — the tick kernel's node pass and the push-pull round alike.
// Refutation of a leave intent about ourselves: serf/base.rs:1470-1480 → broadcast_join(clock.time()), :381-397
SFS_HD void refute_leave(Rec& r, u32& clock, u32 limit) {
  const u32 T = clock; witness(clock, T);
  join_intent(r, T, limit);
  r.qjoin = T; r.txj = limit;
}
// A buffered intent that changed gets the tick as its wall time: NodeIntent.wall_time (types/member.rs:32)
SFS_HD void stamp_intent(Rec& r, const Words& before, u32 tick) {
  if (!(r.flags & 1) && r.status != TY_NONE && (r.status != (before.w[6] & 0xff) || r.st != before.w[0])) r.leave_tick = tick + 1;
}
// Is a watcher's own failed probe still a confirmation (its bucket not in the confirmer set, the set not full)?
SFS_HD bool can_confirm(u32 k, u32 mask, u32 v) { return popc(mask) - 1u < k && !(mask & (1u << from_bucket(v))); }
// A watcher of a down subject probes it (wmask: the subjects among the node's neighbours).
SFS_HD bool view_watching(bool watcher, u32 probe_every, u32 down_mask, u32 s, bool self, u32 wmask) {
  return watcher && probe_every && ((down_mask >> s) & 1) && !self && ((wmask >> s) & 1);
}
// The trace's `pending`: queued transmits, or a watcher that has not noticed yet.  Suspect views are counted apart (they sleep).
SFS_HD bool view_pending(const Rec& r, bool watching) {
  return r.mlstate != ML_SUSPECT && (rec_queued(r) || (watching && r.mlstate == ML_ALIVE));
}
// Does the view keep its node awake: queued transmits, or a watcher whose own failed probe may still start or confirm the
// suspicion?  confirm() is can_confirm for this view, asked only of a watched Suspect view.
template <class Confirm>
SFS_HD bool view_awake(const Rec& r, bool watching, Confirm confirm) {
  return rec_queued(r) || (watching && (r.mlstate == ML_ALIVE || (r.mlstate == ML_SUSPECT && confirm())));
}

// Philox4x32-10 (Salmon et al. 2011): the stateless RNG that picks gossip and probe peers,
// keyed (seed) and counted (tick, node, block, domain) so any sharding draws the same edges.
__host__ __device__ inline void philox4x32_10(u32 c0, u32 c1, u32 c2, u32 c3, u32 k0, u32 k1, u32 out[4]) {
  const u32 M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
#ifdef __CUDA_ARCH__
    u32 hi0 = __umulhi(M0, c0), lo0 = M0 * c0, hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
#else
    u64 p0 = (u64)M0 * c0, p1 = (u64)M1 * c2;
    u32 hi0 = (u32)(p0 >> 32), lo0 = (u32)p0, hi1 = (u32)(p1 >> 32), lo1 = (u32)p1;
#endif
    u32 n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += W0; k1 += W1;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
// One uniformly random neighbour slot of a row of `deg` entries (SWIM probe target, push-pull partner).
SFS_HD u32 neighbour_slot(u32 tick, u32 v, u32 domain, u32 seed_lo, u32 seed_hi, u32 deg) {
  u32 w[4];
  philox4x32_10(tick, v, 0, domain, seed_lo, seed_hi, w);
  return ((w[0] & 0xffffu) * deg) >> 16;
}

// Gossip peers of one node for one tick — memberlist kRandomNodes (k uniformly random distinct members
// other than ourselves): m = min(fanout, deg) distinct slots of the node's CSR row, sampled without
// replacement by rank from ONE Philox4x32-10 block (eight 16-bit draws: low half, then high half of words
// 0..3): draw k picks rank j = (h16_k·(deg−k)) >> 16 among the slots not chosen yet; slots pointing at the
// node itself are dropped; peers are used in draw order.  No rejection loop, no divergence, m gathers.
// Every sender draws its peers this way (membership tick, user events, injectors): they ride in the same packets.
constexpr u32 NO_TARGET = 0xffffffffu;
SFS_HD u32 draw16(const u32 (&w)[4], int i) { const u32 x = w[(i >> 1) & 3]; return (i & 1) ? (x >> 16) : (x & 0xffffu); }
// peer_issue draws the slots and requests the neighbour ids (cand[]: col(row0 + slot), loads in flight, v for an unused draw);
// peer_finish drops self slots and packs the targets.
template <int FMAX, class Col>
SFS_HD void peer_issue(u32 tick, u32 v, u32 fanout, u32 seed_lo, u32 seed_hi, u32 row0, u32 deg, Col col, u32 (&cand)[FMAX]) {
  const u32 m = fanout < deg ? fanout : deg;
  u32 w[4];
  philox4x32_10(tick, v, 0, DOMAIN_GOSSIP, seed_lo, seed_hi, w);
  u32 srt[FMAX];                                           // chosen slots so far, ascending; unused entries = NO_TARGET (sort last)
#pragma unroll
  for (int k = 0; k < FMAX; ++k) srt[k] = NO_TARGET;
#pragma unroll
  for (int k = 0; k < FMAX; ++k) {
    u32 j = (draw16(w, k) * (deg - ((u32)k < deg ? (u32)k : deg))) >> 16;
#pragma unroll
    for (int i = 0; i < k; ++i) j += (j >= srt[i]) ? 1u : 0u;         // rank → slot: skip the slots already taken
    const bool use = (u32)k < m;
    const u32 e = row0 + (use ? j : 0u);
    cand[k] = use ? col(e) : v;
    // insert j into the ascending list (only if used): bubble it down from position k
    u32 x = use ? j : NO_TARGET;
#pragma unroll
    for (int i = 0; i < k; ++i) { const u32 lo = srt[i] < x ? srt[i] : x, hi = srt[i] < x ? x : srt[i]; srt[i] = lo; x = hi; }
    srt[k] = x;
  }
}
template <int FMAX>
SFS_HD u32 peer_finish(u32 v, const u32 (&cand)[FMAX], u32 (&tg)[FMAX]) {
  u32 nt = 0;
#pragma unroll
  for (int k = 0; k < FMAX; ++k) tg[k] = NO_TARGET;
#pragma unroll
  for (int k = 0; k < FMAX; ++k) {
    if (cand[k] != v) {                                    // self slots (and the unused tail) are dropped
#pragma unroll
      for (int j2 = 0; j2 <= k; ++j2) tg[j2] = ((u32)j2 == nt) ? cand[k] : tg[j2];
      ++nt;
    }
  }
  return nt;
}

__host__ __device__ inline u32 mulhi32(u32 a, u32 b) {
#ifdef __CUDA_ARCH__
  return __umulhi(a, b);
#else
  return (u32)(((u64)a * b) >> 32);
#endif
}

__host__ __device__ inline u64 mix64(u64 x) {
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ULL;
  x ^= x >> 27; x *= 0x94d049bb133111ebULL;
  x ^= x >> 31; return x;
}
__host__ __device__ inline u64 rec_hash(u64 idx, const Words& x) {
  u64 w0 = x.w[0] | ((u64)x.w[1] << 32), w1 = x.w[2] | ((u64)x.w[3] << 32), w2 = x.w[4] | ((u64)x.w[5] << 32), w3 = x.w[6] | ((u64)x.w[7] << 32);
  return mix64(w0 ^ mix64(w1 ^ mix64(w2 ^ mix64(w3 ^ mix64(idx + 0x9e3779b97f4a7c15ULL)))));
}
__host__ __device__ inline u64 node_hash(u64 idx, u64 ns) {
  const u64 w = node_word(nw_clock(ns), nw_up(ns), nw_sstate(ns));
  return mix64(w ^ mix64(idx + 0x9e3779b97f4a7c15ULL));
}

}  // namespace sfs
