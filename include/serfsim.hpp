// serfsim.hpp — header-only C++ host layer above the C ABI (include/serfsim.h).
//
// The reference's host code is Rust; with no Rust toolchain in this environment the host side that a
// maintainer would write above the FFI is given here in C++17, with the reference's names and argument meaning:
//
//   serf::MemberStatus            ↔ serf-core/src/types/member.rs:54-113 (same u8 codes, same as_str())
//   serf::LamportTime             ↔ serf-core/src/types/clock.rs:14
//   serf::Options                 ↔ serf-core/src/options.rs (the memberlist LAN profile it embeds, :521)
//   serf::Serf::join/leave/remove_failed_node/members/stats/shutdown
//                                    ↔ serf-core/src/serf/api.rs:318-361, 422-499, 505-515, 136-146, 150-183
//   serf::Serf::user_event         ↔ serf-core/src/serf/api.rs:241-299
//   serf::MemberEventType, EventSubscriber-style callback
//                                    ↔ serf-core/src/event.rs:325-328, serf/delegate.rs:557-582
//
// A `Serf` here is a whole simulated cluster; the node an operation originates from is an explicit argument.
// Errors are values in the reference (`Result<_, Error>`, error.rs); here every failing C call throws
// serf::Error carrying the ABI code and serfsim_last_error().
#pragma once
#include <cstdint>
#include <functional>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "serfsim.h"

namespace serf {

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& what) : std::runtime_error("serfsim error " + std::to_string(c) + ": " + what), code(c) {}
};
inline int check(int rc) {
  if (rc < 0) throw Error(rc, serfsim_last_error());
  return rc;
}

// types/member.rs:54-113
enum class MemberStatus : uint8_t { None = 0, Alive = 1, Leaving = 2, Left = 3, Failed = 4 };
inline const char* as_str(MemberStatus s) {          // MemberStatus::as_str, types/member.rs:96-107
  switch (s) {
    case MemberStatus::None: return "none";
    case MemberStatus::Alive: return "alive";
    case MemberStatus::Leaving: return "leaving";
    case MemberStatus::Left: return "left";
    case MemberStatus::Failed: return "failed";
  }
  return "unknown";
}
enum class MemberEventType : uint32_t { Join = 0, Leave = 1, Failed = 2, Update = 3, Reap = 4 };   // event.rs:325-328

using LamportTime = uint64_t;                         // types/clock.rs:14

// options.rs:495-530 + MemberlistOptions::lan() (:521), in gossip ticks
struct Options {
  serfsim_config_t c;
  Options() { serfsim_default_config(&c); }
  Options& with_nodes(uint32_t n) { c.n_nodes = n; return *this; }
  Options& with_tracked_subjects(uint32_t r) { c.slots = r; return *this; }
  Options& with_gossip_nodes(uint32_t f) { c.fanout = f; return *this; }                 // memberlist gossip_nodes
  Options& with_retransmit_mult(uint32_t m) { c.retransmit_mult = m; return *this; }
  Options& with_suspicion_mult(uint32_t m) { c.suspicion_mult = m; return *this; }
  Options& with_suspicion_max_timeout_mult(uint32_t m) { c.suspicion_max_timeout_mult = m; return *this; }
  Options& with_probe_interval_ticks(uint32_t t) { c.probe_interval_ticks = t; return *this; }
  Options& with_push_pull_interval_ticks(int32_t t) { c.push_pull_interval_ticks = t; return *this; }
  Options& with_reap_interval_ticks(uint32_t t) { c.reap_interval_ticks = t; return *this; }            // options.rs:506
  Options& with_tombstone_timeout_ticks(uint32_t t) { c.tombstone_timeout_ticks = t; return *this; }    // :509
  Options& with_reconnect_timeout_ticks(uint32_t t) { c.reconnect_timeout_ticks = t; return *this; }    // :508
  Options& with_recent_intent_timeout_ticks(uint32_t t) { c.recent_intent_timeout_ticks = t; return *this; }   // :515
  Options& with_seed(uint64_t s) { c.seed = s; return *this; }
  Options& with_device(int32_t d) { c.device = d; return *this; }
  Options& with_trace(bool on) { c.trace = on ? 1u : 0u; return *this; }
};

// serf/api.rs:588-602 (Stats) + the simulator's dissemination counters
using Stats = serfsim_stats_t;

class Serf {
 public:
  // Serf::new (serf/base.rs:62-344): one handle = the whole cluster on the GPU
  explicit Serf(const Options& opts) : n_(opts.c.n_nodes), slots_(opts.c.slots) { check(serfsim_create(&opts.c, &h_)); }
  Serf(const Serf&) = delete;
  Serf& operator=(const Serf&) = delete;
  Serf(Serf&& o) noexcept : h_(o.h_), n_(o.n_), slots_(o.slots_), cb_(std::move(o.cb_)) { o.h_ = nullptr; }
  ~Serf() { shutdown(); }

  // Serf::shutdown (serf/api.rs:517-584): releases the device state
  void shutdown() { if (h_) { serfsim_destroy(h_); h_ = nullptr; } }

  // the member list peers are drawn from (memberlist's node list): CSR over node ids
  void set_topology(const std::vector<uint64_t>& row_ptr, const std::vector<uint32_t>& col_idx) {
    if (row_ptr.size() != (size_t)n_ + 1 || col_idx.size() != row_ptr.back()) throw Error(SERFSIM_E_INVAL, "CSR shape mismatch");
    check(serfsim_set_topology_csr(h_, row_ptr.data(), col_idx.data()));
  }
  void track(const std::vector<uint32_t>& subjects) {
    if (subjects.size() != slots_) throw Error(SERFSIM_E_INVAL, "one subject per tracked slot");
    check(serfsim_set_subjects(h_, subjects.data()));
  }

  // Serf::join (serf/api.rs:318-361) at `node`, effective at gossip tick `tick`
  void join(uint32_t node, uint32_t tick = 0) { check(serfsim_inject(h_, tick, SERFSIM_OP_JOIN, node, 0)); }
  // Serf::leave (serf/api.rs:422-499)
  void leave(uint32_t node, uint32_t tick = 0) { check(serfsim_inject(h_, tick, SERFSIM_OP_LEAVE, node, 0)); }
  // Serf::remove_failed_node (serf/api.rs:505-515 → force_leave, serf/base.rs:454-480): `origin` asks the cluster to forget subject `slot`
  void remove_failed_node(uint32_t origin, uint32_t slot, uint32_t tick = 0) { check(serfsim_inject(h_, tick, SERFSIM_OP_FORCE_LEAVE, origin, slot)); }
  /// Serf::remove_failed_node_prune (serf/api.rs:513): the leave intent carries `prune`, receivers erase the member
  void remove_failed_node_prune(uint32_t origin, uint32_t slot, uint32_t tick = 0) { check(serfsim_inject(h_, tick, SERFSIM_OP_FORCE_LEAVE_PRUNE, origin, slot)); }
  // fault injection (cf. MessageDropper, serf/delegate.rs:42-45)
  void fail(uint32_t node, uint32_t tick = 0) { check(serfsim_inject(h_, tick, SERFSIM_OP_FAIL, node, 0)); }
  void rejoin(uint32_t node, uint32_t tick = 0) { check(serfsim_inject(h_, tick, SERFSIM_OP_REJOIN, node, 0)); }

  // Serf::user_event (serf/api.rs:241-299): declare the tracked events once, then fire event `event` at `origin`
  void track_user_events(const std::vector<uint32_t>& content_ids) { check(serfsim_set_user_events(h_, (uint32_t)content_ids.size(), content_ids.data())); }
  void user_event(uint32_t origin, uint32_t event, uint32_t tick = 0) { check(serfsim_inject(h_, tick, SERFSIM_OP_USER_EVENT, origin, event)); }
  // which nodes handed the event to their EventSubscriber (event.rs:396-512)
  std::vector<uint8_t> user_event_seen(uint32_t event) const { std::vector<uint8_t> v(n_); check(serfsim_user_event_seen(h_, event, v.data())); return v; }
  std::vector<LamportTime> event_time() const { std::vector<LamportTime> v(n_); check(serfsim_event_time(h_, v.data())); return v; }
  serfsim_uevent_stats_t user_event_stats() const { serfsim_uevent_stats_t s; check(serfsim_user_event_stats(h_, &s)); return s; }
  // the (name, payload) bytes of every tracked event, after track_user_events: push-pull messages then carry the event ring
  void user_event_content(const std::vector<std::string>& names, const std::vector<std::string>& payloads) {
    if (names.size() != payloads.size()) throw Error(SERFSIM_E_INVAL, "one name and one payload per tracked event");
    std::vector<const uint8_t*> np, pp;
    std::vector<size_t> nl, pl;
    for (size_t e = 0; e < names.size(); ++e) {
      np.push_back((const uint8_t*)names[e].data()); nl.push_back(names[e].size());
      pp.push_back((const uint8_t*)payloads[e].data()); pl.push_back(payloads[e].size());
    }
    check(serfsim_set_user_event_content(h_, (uint32_t)names.size(), np.data(), nl.data(), pp.data(), pl.data()));
  }
  // SerfDelegate::local_state (serf/delegate.rs:386-425) of nodes [first, first + count): the bytes and count + 1 offsets
  std::pair<std::vector<uint8_t>, std::vector<uint64_t>> local_state(uint32_t first, uint32_t count) const {
    std::vector<uint64_t> off((size_t)count + 1);
    size_t total = 0;
    serfsim_wire_local_state_range(h_, first, count, nullptr, 0, off.data(), &total);      // sizing call
    std::vector<uint8_t> bytes(total ? total : 1);
    check(serfsim_wire_local_state_range(h_, first, count, bytes.data(), bytes.size(), off.data(), &total));
    bytes.resize(total);
    return {std::move(bytes), std::move(off)};
  }

  // the hot path
  void step(uint32_t ticks = 1) { check(serfsim_step(h_, ticks)); }
  // returns {convergence step count, converged?}
  std::pair<uint32_t, bool> run_until_converged(uint32_t max_ticks) {
    uint32_t t = 0;
    const int rc = check(serfsim_run_until_converged(h_, max_ticks, &t));
    return {t, rc == 0};
  }

  // Serf::members (serf/api.rs:136-146): status of subject `slot` as seen by every node
  std::vector<MemberStatus> members(uint32_t slot = 0) const {
    std::vector<uint8_t> raw(n_);
    check(serfsim_member_status(h_, slot, raw.data()));
    std::vector<MemberStatus> out(n_);
    for (size_t i = 0; i < raw.size(); ++i) out[i] = static_cast<MemberStatus>(raw[i]);
    return out;
  }
  std::vector<LamportTime> status_ltime(uint32_t slot = 0) const { std::vector<LamportTime> v(n_); check(serfsim_status_ltime(h_, slot, v.data())); return v; }
  // the same vector as the device keeps it (u32; a run that would leave that range fails with SERFSIM_E_OVERFLOW): half the bytes over PCIe
  std::vector<uint32_t> status_ltime_u32(uint32_t slot = 0) const { std::vector<uint32_t> v(n_); check(serfsim_status_ltime_u32(h_, slot, v.data())); return v; }
  std::vector<uint32_t> lamport_time_u32() const { std::vector<uint32_t> v(n_); check(serfsim_lamport_time_u32(h_, v.data())); return v; }
  // LamportClock::time of every node (types/clock.rs:142)
  std::vector<LamportTime> lamport_time() const { std::vector<LamportTime> v(n_); check(serfsim_lamport_time(h_, v.data())); return v; }
  // Serf::stats (serf/api.rs:150-183)
  Stats stats() const { Stats s; check(serfsim_stats(h_, &s)); return s; }

  // EventDelegate / EventSubscriber (serf/delegate.rs:557-582, event.rs:396-512): batched member events between steps
  using EventHandler = std::function<void(uint32_t tick, MemberEventType, const std::vector<uint32_t>& ids)>;
  void subscribe(EventHandler fn) {
    cb_ = std::move(fn);
    check(serfsim_set_event_cb(h_, &Serf::trampoline, this));
  }

  serfsim_t* raw() const { return h_; }

 private:
  static void trampoline(void* user, uint32_t tick, uint32_t type, const uint32_t* ids, uint32_t n) {
    auto* self = static_cast<Serf*>(user);
    if (self->cb_) self->cb_(tick, static_cast<MemberEventType>(type), std::vector<uint32_t>(ids, ids + n));
  }
  serfsim_t* h_ = nullptr;
  uint32_t n_, slots_;
  EventHandler cb_;
};

}  // namespace serf
