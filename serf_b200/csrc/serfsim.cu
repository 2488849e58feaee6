// serfsim.cu — host side of the simulator and its C ABI (include/serfsim.h).
//
// The reference's host code is Rust; Rust is not available in this build environment, so the
// host layer above the C ABI is C++ and mirrors the reference's names: Options/MemberlistOptions
// fields (serf-core/src/options.rs:495-530), Serf::{join,leave,remove_failed_node,members,stats}
// (serf/api.rs), MemberStatus (types/member.rs:54-58), MemberEventType (event.rs:325-328).
// Device memory, streams and the per-tick launch sequence live here; the kernels are in
// tick_kernel.cu.  There is no CPU execution path: without a CUDA device every entry point fails.
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <optional>
#include <string>
#include <unordered_set>
#include <vector>

#include "../../include/serfsim.h"
#include "owned.cuh"
#include "tick_kernel.cuh"
#include "wire.cuh"

using namespace sfs;

// The kernels index a tick's trace row by ROW_* (tick_kernel.cuh); the host hands it out as serfsim_tick_row_t.
#define SFS_ROW_FIELD(i, f) static_assert(i == offsetof(serfsim_tick_row_t, f) / sizeof(uint64_t), #i " is serfsim_tick_row_t::" #f)
SFS_ROW_FIELD(ROW_PACKETS, packets); SFS_ROW_FIELD(ROW_EDGES, edge_updates); SFS_ROW_FIELD(ROW_MESSAGES, messages); SFS_ROW_FIELD(ROW_CHANGED, changed);
SFS_ROW_FIELD(ROW_PENDING, pending); SFS_ROW_FIELD(ROW_EVENTS, events); SFS_ROW_FIELD(ROW_SUSPECTS, suspects); SFS_ROW_FIELD(ROW_HASH, hash);
#undef SFS_ROW_FIELD
static_assert(sizeof(serfsim_tick_row_t) == ROW_FIELDS * sizeof(uint64_t), "a trace row is ROW_FIELDS counters");

namespace {

thread_local std::string g_err;

int fail(int code, const std::string& msg) { g_err = msg; return code; }

struct HostOp { u32 tick, op, node, slot; u64 seq; };

// memberlist retransmit limit: retransmit_mult * ceil(log10(n + 1))  [external crate, restated].  In 64 bits: serfsim_create
// rejects a product outside 1..255 (the budgets are u8) instead of letting it wrap in u32.
u64 retransmit_limit(u32 mult, u64 n) {
  u64 digits = 0;
  u64 p = 1;
  while (p < n + 1) { p *= 10; ++digits; }
  return (u64)mult * digits;
}

// Bounds of the configuration's numeric range (serfsim.h, DESIGN §2 rule 10).
//  - Suspicion timeouts: at most 2^30 ticks.  A run stores a 64-byte trace row per tick, so no device holds 2^31 ticks of one
//    run; tick + timeout and the confirmation update deadline - timeout[c] + timeout[c+1] then stay below 2^31 + 2^30, inside u32
//    and never 0 ("no timer").  2^30 ticks are 6.8 years at 200 ms per tick.
//  - Bootstrap Lamport times (init_clock, init_status_ltime): below LTIME_LIMIT - 16, so the bootstrap state is representable
//    and a run starts at least 16 Lamport increments away from SERFSIM_E_OVERFLOW.
constexpr u64 TIMEOUT_LIMIT_TICKS = 1ull << 30;
constexpr u32 INIT_LTIME_BOUND = LTIME_LIMIT - 16;

const char* const kTimeoutTooLong =
    "suspicion timeout longer than 2^30 ticks (suspicion_mult, suspicion_max_timeout_mult, probe_interval_ticks, gossip_interval_ms)";

// The integer (ms) part of suspicion_table in exact 128-bit arithmetic: null when every intermediate fits in int64 and the
// exact timeouts are at most TIMEOUT_LIMIT_TICKS, else the reason.  The entries lie between ceil(min_ms / tick_ms) and
// ceil(max(min_ms, max_ms) / tick_ms) (just the former when k < 1), so that bounds them all (up to the rounding of the double step,
// which serfsim_create checks on the table itself).  Only a config that passes this is given to suspicion_table.
const char* suspicion_table_unrepresentable(u32 susp_mult, u32 max_mult, u32 probe_ticks, u32 tick_ms, u64 n) {
  const double node_scale = std::max(1.0, std::log10(std::max(1.0, (double)n)));
  const __int128 i64max = (__int128)INT64_MAX;
  const __int128 interval_ms = (__int128)probe_ticks * tick_ms;
  const __int128 prod = (__int128)susp_mult * (int64_t)(node_scale * 1000.0) * interval_ms;
  if (interval_ms > i64max || prod > i64max) return "suspicion timeout: suspicion_mult x probe_interval_ticks x gossip_interval_ms overflows the 64-bit ms arithmetic";
  const __int128 min_ms = prod / 1000, max_ms = (__int128)max_mult * min_ms;
  if (max_ms > i64max) return "suspicion timeout: suspicion_max_timeout_mult x the minimum timeout overflows the 64-bit ms arithmetic";
  const bool confirmations = (int64_t)susp_mult - 2 >= 1 && (int64_t)n - 2 >= (int64_t)susp_mult - 2;   // k >= 1: max_ms is used
  const __int128 top = confirmations ? std::max(min_ms, max_ms) : min_ms;
  if ((top + tick_ms - 1) / tick_ms > (__int128)TIMEOUT_LIMIT_TICKS) return kTimeoutTooLong;
  return nullptr;
}

// memberlist suspicion timeouts (Lifeguard), in ticks  [external crate, restated]:
//   min = suspicion_mult · max(1, log10 n) · probe_interval, max = suspicion_max_timeout_mult · min,
//   k = suspicion_mult − 2 (0 if n − 2 < k), timeout(c) = max − log(c+1)/log(k+1)·(max − min) ≥ min.
// The only floating point on the whole path; it runs once on the host and yields integers.
std::vector<u32> suspicion_table(u32 susp_mult, u32 max_mult, u32 probe_ticks, u32 tick_ms, u64 n) {
  const double node_scale = std::max(1.0, std::log10(std::max(1.0, (double)n)));
  const int64_t interval_ms = (int64_t)probe_ticks * tick_ms;
  const int64_t min_ms = (int64_t)susp_mult * (int64_t)(node_scale * 1000.0) * interval_ms / 1000;
  const int64_t max_ms = (int64_t)max_mult * min_ms;
  int64_t k = (int64_t)susp_mult - 2;
  if ((int64_t)n - 2 < k) k = 0;
  if (k < 0) k = 0;
  std::vector<u32> tab;
  for (int64_t c = 0; c <= k; ++c) {
    int64_t ms = min_ms;
    if (k >= 1) {
      const double frac = std::log((double)c + 1.0) / std::log((double)k + 1.0);
      ms = (int64_t)std::floor((double)max_ms - frac * (double)(max_ms - min_ms));
      if (ms < min_ms) ms = min_ms;
    }
    int64_t ticks = (ms + tick_ms - 1) / tick_ms;
    if (ticks < 1) ticks = 1;
    tab.push_back((u32)ticks);
  }
  return tab;
}

// Run-time switches: every SERFSIM_* environment variable the library reads, read once per handle by read_switches (serfsim_create).
// Defaults are the measured-fastest settings; the switches exist for A/B measurements and debugging and never change results.
struct Switches {
  int gridmul = 2;            // SERFSIM_GRIDMUL >= 1 (else 2): waves of resident CTAs in the tick kernels' persistent grid
  bool minb5 = false;         // SERFSIM_MINB=5: single-slot runs size their grid for 5 CTAs/SM, and unsharded ones launch the 5-CTA instance
  bool tma = false;           // SERFSIM_TMA=1: single-slot runs stage tiles through the TMA pipeline if a tile's CSR span fits 48 KB
  bool tma_sync = false;      // SERFSIM_TMA_SYNC=1: the TMA pipeline's barrier-synchronised form
  bool udeg = true;           // SERFSIM_UDEG=0: row offsets are loaded even when every row has the same degree (the general path)
  u32 ahead = 1;              // SERFSIM_AHEAD=0|1|2: multi-slot kernel requests one tile ahead off / in saturated ticks / always
  u32 sv = 1;                 // SERFSIM_SV=0|1|2: multi-slot ticks as per-view passes (sharded: single-view dual launch) off / on / check mode
  bool compact = true;        // SERFSIM_COMPACT=0: tile-by-tile walk in unsaturated ticks too
  bool dedup = true;          // SERFSIM_DEDUP=0: unsharded sends issue every RED, also those that change nothing
  bool no_skip = false;       // SERFSIM_NO_SKIP=1: process every tile, every view, every tick
  bool no_jump = false;       // SERFSIM_NO_JUMP (set): the convergence loop launches the ticks the cluster sleeps through
  u32 chunk = 0;              // SERFSIM_CHUNK=n (>= 1): ticks per launch chunk; 0 (unset): 8, doubling up to 32, 8 again after a jump
  double win_factor = 1.25;   // SERFSIM_WIN_FACTOR=x: sharded receive windows hold x times the expected entries per tick and peer
  bool no_fuse = false;       // SERFSIM_NO_FUSE (set): sharded ticks launch a separate publish kernel instead of the fused one
  int l2_persist = 0;         // SERFSIM_L2_PERSIST != 0: set aside the largest persisting L2 carve-out (off: it takes L2 from every plane)
  bool l2_window = false;     // SERFSIM_L2_WINDOW=1: stream access-policy window over the inbox being written
  bool verbose = false;       // SERFSIM_VERBOSE (set): print the L2 limits and the tick kernel and grid picked for each topology
  bool debug_loop = false;    // SERFSIM_DEBUG_LOOP (set): print the convergence loop's state after every launch chunk
  bool xtiming = false;       // SERFSIM_XTIMING (set): serfsim_destroy prints the tick kernel / exchange split of a timed sharded run
};

Switches read_switches() {
  auto num = [](const char* name, int dflt) { const char* e = getenv(name); return e ? atoi(e) : dflt; };
  auto set = [](const char* name) { return getenv(name) != nullptr; };
  Switches s;
  s.gridmul = num("SERFSIM_GRIDMUL", s.gridmul); if (s.gridmul < 1) s.gridmul = 2;
  s.minb5 = num("SERFSIM_MINB", 0) == 5;
  s.tma = num("SERFSIM_TMA", s.tma) != 0;
  s.tma_sync = num("SERFSIM_TMA_SYNC", s.tma_sync) != 0;
  s.udeg = num("SERFSIM_UDEG", s.udeg) != 0;
  s.ahead = (u32)std::min(2, std::max(0, num("SERFSIM_AHEAD", s.ahead)));
  s.sv = (u32)std::min(2, std::max(0, num("SERFSIM_SV", s.sv)));
  s.compact = num("SERFSIM_COMPACT", s.compact) != 0;
  s.dedup = num("SERFSIM_DEDUP", s.dedup) != 0;
  s.no_skip = num("SERFSIM_NO_SKIP", s.no_skip) != 0;
  s.no_jump = set("SERFSIM_NO_JUMP");
  s.chunk = set("SERFSIM_CHUNK") ? (u32)std::max(1, num("SERFSIM_CHUNK", 1)) : 0u;
  if (const char* e = getenv("SERFSIM_WIN_FACTOR")) s.win_factor = atof(e);
  s.no_fuse = set("SERFSIM_NO_FUSE");
  s.l2_persist = num("SERFSIM_L2_PERSIST", s.l2_persist);
  s.l2_window = num("SERFSIM_L2_WINDOW", s.l2_window) != 0;
  s.verbose = set("SERFSIM_VERBOSE");
  s.debug_loop = set("SERFSIM_DEBUG_LOOP");
  s.xtiming = set("SERFSIM_XTIMING");
  return s;
}

}  // namespace

struct serfsim {
  serfsim_config_t cfg{};
  u32 N = 0, R = 0, first = 0, count = 0, shard_size = 0;
  u32 stride = 0;                  // count rounded up to a whole 256-node tile: stride of every per-slot plane
  Rules rules{};
  Stream stream;                   // declared before every buffer: destroyed after them
  Event ev0, ev1;
  // device state
  DevArray<uint4> d_rec;           // [R][stride] × 32 B (transmit-budget bytes zero)
  DevArray<u32> d_qword;           // [R][stride] queue words (transmit budgets)
  DevArray<u32> d_inbox[2];        // [3][R][stride]
  DevArray<u64> d_node;            // [stride]
  DevArray<u8> d_busy;             // [stride] per-node busy byte
  DevArray<u16> d_watch;           // [stride] per-node watcher mask (subjects among the node's neighbours)
  bool watch_dirty = true;
  DevArray<uint4> d_snap_rec;      // push-pull rounds (allocated by serfsim_create): end-of-tick snapshot of the records …
  DevArray<u64> d_snap_node;       // … and of the node words
  DevArray<const uint4*> d_peer_snap_rec;   // sharded push-pull: device arrays of every rank's snapshot pointers
  DevArray<const u64*> d_peer_snap_node;
  DevArray<u8> d_hot[2];                  // [n_tiles] per tick parity
  DevArray<u8> d_hot_static;              // [n_tiles] tiles that hold a watcher (never consumed)
  DevArray<u32> d_node_due;               // [stride] per-node earliest suspicion deadline (tick_kernel.cuh)
  DevArray<u32> d_carry;                  // [stride] per-view passes: carry words (tick_kernel.cuh: CARRY_*); unsharded multi-slot runs only
  DevArray<u32> d_tile_due;               // [n_tiles] earliest suspicion deadline of a tile's nodes (the timer wheel)
  DevArray<u32> d_sched;                  // scheduler words (tick_kernel.cuh: SCHED_*)
  u32 n_tiles = 0;
  DevArray<u32> d_rowptr;          // [stride+8]
  DevArray<u32> d_col;
  DevArray<u32> d_ev_node, d_ev_op, d_ev_slot;
  size_t ev_cap = 0;
  DevArray<u64> d_trace;           // [trace_cap][8]
  DevArray<u32> d_kinds;           // [trace_cap+1][4]; row t+1 = messages by kind sent in tick t
  DevArray<u32> d_view_kinds;      // [trace_cap+1][R][4]; row t+1 = messages by view and kind sent in tick t by per-view passes (zero otherwise)
  u32 trace_cap = 0;
  MappedWords pin_overflow;        // written by kernels on the rare error paths, read by the host without a copy
  u32* d_overflow = nullptr;       // its device address
  DevArray<u32> d_subj;
  DevArray<u64> d_scratch;         // summary / hash output
  DevArray<u64> d_stage;           // getter staging, count × 8 B
  // user events (SURVEY §8f row 3), allocated together by serfsim_set_user_events: [stride] 16-byte event records and arrived-event
  // masks per tick parity, [MAX_UEVENTS] Lamport times, [8] totals; push-pull rounds: the record snapshot partners read, and every rank's
  struct UserEvents { DevArray<uint4> state, snap; DevArray<u32> inbox[2], ltime; DevArray<u64> totals; DevArray<const uint4*> peer_snap; };
  std::optional<UserEvents> ue;
  UeTable ue_table{};              // n = 0: user events off
  wire::UeWire ue_wire{};          // wire form of the tracked events (serfsim_set_user_event_content); n = 0: none
  DevArray<u8> d_ue_entries;       // its UserEvents.events entries on the device
  u32 ue_injected = 0;             // tracked events already scheduled (each may be injected once)
  u32 ue_origin[MAX_UEVENTS] = {0};
  u32 ue_fire_tick[MAX_UEVENTS] = {0};  // origin node of each scheduled event (its shard is the one that stamps the Lamport time)
  // byzantine injectors (BASELINE configs[4]): allocated by serfsim_set_byzantine (sharded runs: by serfsim_create, peers raise the
  // flags): [stride] sender flags, [4] totals, [byz_n] ascending ids
  u32 byz_n = 0, byz_delta = 2;    // byz_n: injectors of THIS shard
  bool byz_on = false;             // any injector anywhere (all ranks agree): changes the convergence rule and the drain kernel
  struct Injectors { DevArray<u8> anomaly; DevArray<u64> totals; DevArray<u32> ids; };
  std::optional<Injectors> byz;
  DevArray<u8*> d_peer_anomaly;    // sharded runs: device array of every rank's flag array
  // host state
  std::vector<HostOp> ops;         // sorted by (tick, seq)
  std::unordered_set<u64> op_keys; // (tick << 32 | node): at most one operation per node per tick
  bool ops_dirty = false;
  u64 op_seq = 0;
  std::vector<u32> subj;
  u32 up_mask = 0;
  u32 ever_down = 0;               // subjects that have been down at some tick since the reset (only those are probed, suspected, run timers)
  int grid_sv = 0;                 // grid of the single-view kernel
  u32 tick = 0;
  bool has_topo = false;
  u32 stage_col_bytes = 0;         // 0: direct-load kernel; else bytes of CSR per TMA stage
  u32 max_tile_edges = 0;          // largest 16-byte-aligned CSR span of one 256-node tile (sizes the TMA stage)
  u32 udeg = 0;                    // uniform out-degree of the shard's rows (0: degrees differ)
  std::vector<serfsim_tick_row_t> rows;   // rows pulled from the device so far (global sums when sharded)
  // device-side convergence gate (tick_kernel.cuh: Gate)
  DevArray<u32> d_runctl;          // [0] done flag, [1] first quiescent tick
  MappedWords pin_ctl;             // [4] the verdict, written by the gate's leader thread and read once per chunk
  u32* d_pin_ctl = nullptr;        // its device address
  DevArray<u64> d_grow;            // sharded runs: [trace_cap][8] global trace rows, summed on the device by the drain kernel
  bool gate_on = false;
  u32 gate_first = 0;              // first tick of the current run_until_converged call (it always runs)
  std::vector<u32> launch_log;     // kernels launched per tick since the timing window opened (ticks past the quiescent one do not count)
  u32 launch_log_first = 0;
  bool timing_open = false;
  double last_ms = 0.0;
  u64 last_launches = 0, launches = 0;
  serfsim_event_cb cb = nullptr;
  void* cb_user = nullptr;
  std::vector<u8> reported;        // last status reported per slot
  int grid = 1;
  int ctas_per_sm = 4;             // resident CTAs per SM the membership kernel's grid is sized for (and its __launch_bounds__ instance)
  int sms = 132;                   // the device's SM count
  Switches sw;                     // run-time switches, read at serfsim_create
  // multi-GPU
  DevArray<u64> d_win_data[2];                 // my receive windows [parity][world][win_cap]  (IPC-exported)
  DevArray<u32> d_ctrl;                        // my control block [parity][counts[8] | flags[8]] (IPC-exported)
  DevArray<u32> d_send_count;                  // [world] entries written into each peer's window this tick
  DevArray<u64*> d_peer_data[2];               // device arrays of peer window pointers, per parity
  DevArray<u32*> d_peer_ctrl;                  // device array of peer control-block pointers
  u32 xepoch = 0;                              // executed-tick counter of the exchange (never rewinds): stamps and parity
  u32 win_cap = 0;
  u32 win_cap_base = 0;                        // capacity sized for the membership entries alone (serfsim_create)
  bool connected = false;
  bool loopback = false;                       // serfsim_comm_loopback: profiling aid, the handle exchanges with itself
  serfsim_barrier_fn barrier = nullptr; serfsim_allreduce_u64_fn allreduce = nullptr; void* comm_user = nullptr;
  std::vector<IpcMapping> ipc_opened;
  bool tick_timing = false;
  size_t l2_persist_max = 0, l2_window_max = 0;
  // asynchronous result read-back (serfsim_results_async): extraction into a ring of staging buffers on the launch stream,
  // device→host copies on a second stream so that they overlap the ticks of the caller's next step
  struct ResBuf { DevArray<unsigned char> d; Event copied; bool used = false; };
  struct ReadBack { Stream copy_stream; Event extracted; ResBuf res[4]; u32 next = 0; };
  std::optional<ReadBack> rb;      // allocated together by the first serfsim_results_async
  std::vector<Event> tick_ev;      // 2 per tick when tick_timing
  std::vector<Event> mid_ev;       // after the tick kernel (multi-GPU breakdown, SERFSIM_XTIMING=1)
};

namespace {

int slot_of(const serfsim* h, u32 node) {
  for (u32 s = 0; s < h->R; ++s) if (h->subj[s] == node) return (int)s;
  return -1;
}

int ensure_trace(serfsim* h, u32 need) {
  if (need <= h->trace_cap) return 0;
  u32 cap = std::max<u32>(1024, h->trace_cap);
  while (cap < need) cap *= 2;
  CU(h->d_trace.grow((size_t)cap * ROW_FIELDS, h->stream));
  CU(h->d_kinds.grow(((size_t)cap + 1) * 4, h->stream));
  CU(h->d_view_kinds.grow(((size_t)cap + 1) * h->R * 4, h->stream));
  if (h->cfg.world_size > 1) CU(h->d_grow.grow((size_t)cap * ROW_FIELDS, h->stream));
  h->trace_cap = cap;
  return 0;
}

int upload_ops(serfsim* h) {
  if (!h->ops_dirty) return 0;
  std::stable_sort(h->ops.begin(), h->ops.end(), [](const HostOp& a, const HostOp& b) { return a.tick != b.tick ? a.tick < b.tick : a.seq < b.seq; });
  const size_t n = h->ops.size();
  if (n > h->ev_cap) {
    size_t cap = std::max<size_t>(1024, h->ev_cap);
    while (cap < n) cap *= 2;
    CU(h->d_ev_node.alloc(cap)); CU(h->d_ev_op.alloc(cap)); CU(h->d_ev_slot.alloc(cap));
    h->ev_cap = cap;
  }
  if (n) {
    std::vector<u32> a(n), b(n), c(n);
    for (size_t i = 0; i < n; ++i) { a[i] = h->ops[i].node; b[i] = h->ops[i].op; c[i] = h->ops[i].slot; }
    CU(cudaMemcpyAsync(h->d_ev_node, a.data(), n * 4, cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_ev_op, b.data(), n * 4, cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_ev_slot, c.data(), n * 4, cudaMemcpyHostToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));     // staging vectors die here
  }
  h->ops_dirty = false;
  return 0;
}

bool future_ops(const serfsim* h, u32 after_tick) {       // any op scheduled at tick > after_tick
  return !h->ops.empty() && h->ops.back().tick > after_tick;
}

// The host operations of tick t: ops[begin, end) (ops is sorted by tick).
struct OpRange { u32 begin, end; };
OpRange ops_of_tick(const serfsim* h, u32 t) {
  auto lo = std::lower_bound(h->ops.begin(), h->ops.end(), t, [](const HostOp& o, u32 tt) { return o.tick < tt; });
  auto hi = std::upper_bound(lo, h->ops.end(), t, [](u32 tt, const HostOp& o) { return tt < o.tick; });
  return {(u32)(lo - h->ops.begin()), (u32)(hi - h->ops.begin())};
}
bool ops_at(const serfsim* h, u32 t) { const OpRange r = ops_of_tick(h, t); return r.end > r.begin; }
bool reap_tick(const serfsim* h, u32 t) { return h->cfg.reap_interval_ticks && ((t + 1) % h->cfg.reap_interval_ticks) == 0; }
bool pp_tick(const serfsim* h, u32 t) {         // an anti-entropy round follows tick t
  const u32 pp = (u32)std::max(0, h->cfg.push_pull_interval_ticks);
  return pp && (t + 1) % pp == 0;
}

// How tick t launches its membership kernels (SV_*, tick_kernel.cuh): the one place that decides it.  Multi-slot runs in production mode
// (no trace, no SERFSIM_NO_SKIP, no injectors): unsharded ticks without a host operation or a reaper round run as per-view passes; sharded
// ticks while exactly one subject has ever been down launch the general and the single-view kernel and the device decides (dual launch).
// SERFSIM_SV=2 takes both to the general kernel in check mode.  Call it after the tick's down subjects are in ever_down.
enum class TickRun { General, Passes, Check, Dual };
TickRun tick_run(const serfsim* h, u32 t) {
  if (!h->sw.sv || h->R < 2 || h->R >= 32 || h->cfg.trace || h->sw.no_skip || h->byz_on) return TickRun::General;
  if (h->cfg.world_size > 1) {
    if (__builtin_popcount(h->ever_down) != 1) return TickRun::General;
    return h->sw.sv == 2 ? TickRun::Check : TickRun::Dual;
  }
  if (ops_at(h, t) || reap_tick(h, t) || t + 1 >= CARRY_TICKS) return TickRun::General;
  return h->sw.sv == 2 ? TickRun::Check : TickRun::Passes;
}
// The passes of tick t + 1 choose their loads from their own views' counters of tick t (TickParams::view_kinds_prev) only if every
// inbox write of tick t was a pass's: otherwise (general kernel — host operation, reaper round, trace mode, SERFSIM_SV=0/2 — anti-entropy
// round, injectors, sharded runs) the general kernel's sends and the other writers are not in them, and the passes fall back to the whole
// tick's counters.  Ticks the host jumped over or the device skipped sent nothing: their zero rows are exact either way.  This is the
// one place that decides it.
bool view_kinds_valid(const serfsim* h, u32 t) {
  return tick_run(h, t) == TickRun::Passes && !pp_tick(h, t);          // (injectors: never passes)
}

// The planes as the single-slot kernel sees them: p with every per-slot plane starting at view s, on the single-slot kernel's grid.
TickParams at_view(const serfsim* h, const TickParams& p, u32 s) {
  TickParams q = p;
  q.sv_wshift = s;
  q.rec = p.rec + 2 * (size_t)s * h->stride; q.qword = p.qword + (size_t)s * h->stride;
  q.inbox_rd = p.inbox_rd + (size_t)s * h->stride; q.inbox_wr = p.inbox_wr + (size_t)s * h->stride;
  q.subj[0] = p.subj[s]; q.down_mask = (p.down_mask >> s) & 1u;
  q.tiles_per_cta = (h->n_tiles + h->grid_sv - 1) / h->grid_sv;
  return q;
}

// Timing events, created on first use: ev holds at least n.
int grow_events(std::vector<Event>& ev, size_t n) {
  while (ev.size() < n) { Event e; CU(e.create()); ev.push_back(std::move(e)); }
  return 0;
}

// The tracked user events' Lamport times as the cluster knows them: the origin's shard stamps an event, the other shards may not have it
// yet, so each contributes the stamps of its own nodes' events and every rank gets the sum (a collective when sharded).  Stream idle.
int ue_cluster_ltimes(serfsim* h, u32 lt[MAX_UEVENTS]) {
  CU(cudaMemcpy(lt, h->ue->ltime, h->ue->ltime.bytes(), cudaMemcpyDeviceToHost));
  if (h->cfg.world_size > 1 && h->allreduce) {
    u64 v[MAX_UEVENTS];
    for (u32 e = 0; e < MAX_UEVENTS; ++e) v[e] = (((h->ue_injected >> e) & 1u) && h->ue_origin[e] - h->first < h->count) ? lt[e] : 0;
    h->allreduce(h->comm_user, v, MAX_UEVENTS);
    for (u32 e = 0; e < MAX_UEVENTS; ++e) lt[e] = (u32)v[e];
  }
  return 0;
}

// The summary kernel's output: [0] largest clock, [1] queued intents, [2 + 2s] / [3 + 2s] least / greatest status word of view s.
int read_summary(serfsim* h, std::vector<u64>& out) {
  const u32 nout = 2 + 2 * h->R;
  std::vector<u64> init(nout, 0);
  for (u32 s = 0; s < h->R; ++s) init[2 + 2 * s] = ~0ull;
  out.resize(nout);
  CU(cudaMemcpyAsync(h->d_scratch, init.data(), nout * 8, cudaMemcpyHostToDevice, h->stream));
  launch_summary(h->d_rec, h->d_qword, h->d_node, h->count, h->stride, h->first, h->R, h->d_subj, h->d_scratch, h->stream);
  CU(cudaMemcpyAsync(out.data(), h->d_scratch, nout * 8, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  return 0;
}

// The membership tick's block for tick t with host operations ops[ops.begin, ops.end); the other blocks take their shared fields from it.
TickParams tick_params(const serfsim* h, u32 t, OpRange ops) {
  TickParams p{};
  p.n_local = h->count; p.first = h->first; p.n_global = h->N; p.R = h->R;
  p.fanout = h->cfg.fanout; p.probe_every = h->cfg.probe_interval_ticks; p.tick = t;
  p.down_mask = (~h->up_mask) & ((1u << h->R) - 1);
  p.seed_lo = (u32)h->cfg.seed; p.seed_hi = (u32)(h->cfg.seed >> 32); p.ev_begin = ops.begin; p.ev_end = ops.end;
  p.rules = h->rules;
  for (u32 s = 0; s < h->R; ++s) p.subj[s] = h->subj[s];
  p.rec = h->d_rec; p.qword = h->d_qword; p.inbox_rd = h->d_inbox[(t & 1) ^ 1]; p.inbox_wr = h->d_inbox[t & 1];
  p.node_state = h->d_node; p.busy = h->d_busy; p.watch = h->d_watch; p.row_ptr = h->d_rowptr; p.col = h->d_col;
  p.ev_node = h->d_ev_node; p.ev_op = h->d_ev_op; p.ev_slot = h->d_ev_slot;
  p.row = h->d_trace + (size_t)t * ROW_FIELDS;
  p.kinds_prev = h->d_kinds + (size_t)t * 4;
  p.kinds_cur = h->d_kinds + ((size_t)t + 1) * 4;
  p.overflow = h->d_overflow;
  p.hot_rd = h->d_hot[(t & 1) ^ 1]; p.hot_wr = h->d_hot[t & 1];
  p.stage_col_bytes = h->stage_col_bytes;
  p.reap_now = reap_tick(h, t) ? 1u : 0u;
  p.tombstone_ticks = h->cfg.tombstone_timeout_ticks; p.reconnect_ticks = h->cfg.reconnect_timeout_ticks; p.intent_ticks = h->cfg.recent_intent_timeout_ticks;
  p.stride = h->stride; p.n_tiles = h->n_tiles; p.tiles_per_cta = (h->n_tiles + h->grid - 1) / h->grid;
  p.force_all = (h->cfg.trace != 0) || h->sw.no_skip || p.reap_now;
  p.compact = h->sw.compact ? 1u : 0u;
  p.dedup = h->sw.dedup ? 1u : 0u;
  p.udeg = h->udeg; p.ahead = h->sw.ahead;
  p.tile_due = h->d_tile_due; p.node_due = h->d_node_due; p.hot_static = h->d_hot_static; p.sched = h->d_sched;
  p.sleep_on = (h->sw.no_skip || h->byz_on) ? 0u : 1u;          // injectors send every tick: the cluster never sleeps
  p.pp_every = (u32)std::max(0, h->cfg.push_pull_interval_ticks); p.reap_every = h->cfg.reap_interval_ticks;
  p.host_idle_until = h->d_pin_ctl + 2;
  const bool sharded = h->cfg.world_size > 1;
  const u32 xpar = h->xepoch & 1;
  p.world = (u32)h->cfg.world_size; p.rank = (u32)h->cfg.rank; p.shard_size = h->shard_size; p.win_cap = h->win_cap;
  p.win_data = h->d_peer_data[xpar]; p.send_count = h->d_send_count;
  p.peer_ctrl = h->d_peer_ctrl; p.stamp = h->xepoch + 1; p.xpar = xpar; p.loopback = h->loopback ? 1u : 0u;
  p.fuse_publish = (sharded && !h->byz_on && !h->sw.no_fuse) ? 1u : 0u;
  p.shard_inv = (u32)(0x100000000ull / h->shard_size); p.xcap = p.world > 1 ? XW_TOTAL / (p.world - 1) : 0u;
  if (h->gate_on) {                                // convergence gate: the first kernel of the tick evaluates the row of tick t-1
    const u64* grow = sharded ? h->d_grow : h->d_trace;            // global rows: the device sums them when sharded
    Gate& g = p.gate;
    g.ctl = h->d_runctl; g.host_ctl = h->d_pin_ctl; g.prev_row = t > h->gate_first ? grow + (size_t)(t - 1) * ROW_FIELDS : nullptr; g.tick = t;
    g.future_ops = (t > 0 && future_ops(h, t - 1)) ? 1u : 0u;
    g.pp = p.pp_every; g.byz_on = h->byz_on ? 1u : 0u;
  }
  p.gate.evaluate = h->ue_table.n ? 0u : 1u;       // with user events on, their kernel is the tick's first
  return p;
}

// The user-event tick: it needs the pre-operation up flags and op bits, so it runs first and evaluates the gate.
void launch_user_events(serfsim* h, const TickParams& p) {
  const u32 t = p.tick;
  UeParams u{};
  u.n_local = h->count; u.first = h->first; u.n_global = h->N; u.R = h->R; u.fanout = h->cfg.fanout; u.tick = t;
  u.seed_lo = p.seed_lo; u.seed_hi = p.seed_hi; u.limit = h->rules.limit; u.ev_begin = p.ev_begin; u.ev_end = p.ev_end;
  u.table = h->ue_table; u.state = h->ue->state; u.inbox_rd = h->ue->inbox[(t & 1) ^ 1]; u.inbox_wr = h->ue->inbox[t & 1];
  u.ltime = h->ue->ltime; u.node_state = h->d_node; u.busy = h->d_busy; u.row_ptr = h->d_rowptr; u.col = h->d_col;
  u.ev_node = h->d_ev_node; u.ev_op = h->d_ev_op; u.ev_slot = h->d_ev_slot;
  u.row = p.row; u.totals = h->ue->totals; u.overflow = h->d_overflow; u.sched = h->d_sched;
  u.world = p.world; u.rank = p.rank; u.shard_size = h->shard_size; u.win_cap = h->win_cap;
  u.win_data = p.win_data; u.send_count = h->d_send_count;
  u.gate = p.gate; u.gate.evaluate = 1u;
  launch_uevent(u, h->cfg.trace != 0, h->stream);
  h->last_launches++;
}

// The membership tick as tick_run decides it: the general kernel, per-view passes of the single-slot kernel, or the general kernel and
// the single-view kernel.  p leaves with the fields the launch set (the anti-entropy round takes it as it is).
void launch_membership(serfsim* h, TickParams& p) {
  const u32 t = p.tick;
  const TickRun run = tick_run(h, t);
  if (run != TickRun::General) {
    p.views_host = p.ev_end > p.ev_begin || p.reap_now ? 0xffffffffu : h->ever_down;   // a host operation or a reaper round visits every view
    p.sv_mode = h->sw.sv == 2 ? SV_CHECK : SV_GENERAL;
    p.sv_slot = h->ever_down ? (u32)__builtin_ctz(h->ever_down) : 0u; p.sv_R = h->R;
  }
  if (run == TickRun::Passes) {
    p.sv_mode = SV_PASS; p.carry = h->d_carry;
    p.tiles_per_cta = (h->n_tiles + h->grid_sv - 1) / h->grid_sv;
    const bool own = t > 0 && view_kinds_valid(h, t - 1);
    for (u32 s0 = 0; s0 < h->R; ++s0) {                  // ascending slot order: what the view loop carries from view to view travels through memory
      TickParams q = at_view(h, p, s0);
      q.gate.evaluate = s0 == 0 ? p.gate.evaluate : 0u; q.sv_slot = s0;
      q.view_kinds_prev = own ? h->d_view_kinds + ((size_t)t * h->R + s0) * 4 : p.kinds_prev;
      q.view_kinds_cur = h->d_view_kinds + (((size_t)t + 1) * h->R + s0) * 4;
      launch_tick_pass(q, h->grid_sv, h->stream);
      h->last_launches++;
    }
  } else {
    launch_tick(p, h->cfg.trace != 0, h->grid, h->ctas_per_sm, h->sw.tma_sync, h->stream);
    h->last_launches++;
  }
  if (run == TickRun::Dual) {
    TickParams q = at_view(h, p, p.sv_slot);
    q.sv_mode = SV_SINGLE; q.gate.evaluate = 0u;
    launch_tick_single_view(q, h->grid_sv, h->stream);
    h->last_launches++;
  }
}

// Stale entries of this shard's injectors (before the exchange: peers in other shards get window entries).
void launch_injectors(serfsim* h, const TickParams& p) {
  const u32 t = p.tick;
  ByzParams b{};
  b.n_byz = h->byz_n; b.first = h->first; b.R = h->R; b.stride = h->stride; b.fanout = h->cfg.fanout; b.tick = t;
  b.seed_lo = p.seed_lo; b.seed_hi = p.seed_hi; b.delta = h->byz_delta; b.ids = h->byz->ids; b.rec = h->d_rec; b.node_state = h->d_node;
  b.row_ptr = h->d_rowptr; b.col = h->d_col; b.inbox_wr = h->d_inbox[t & 1]; b.hot_wr = h->d_hot[t & 1]; b.kinds_cur = p.kinds_cur;
  b.anomaly = h->byz->anomaly; b.totals = h->byz->totals;
  b.n_local = h->count; b.world = p.world; b.rank = p.rank; b.shard_size = h->shard_size; b.win_cap = h->win_cap;
  b.win_data = p.win_data; b.send_count = h->d_send_count; b.overflow = h->d_overflow; b.gate = p.gate.ctl;
  launch_byz(b, h->stream);
  h->last_launches++;
}

// The exchange of a sharded tick.  No host round trip: publish (counts + flag into every peer's control block) and drain (waits for the
// peers' flags of this exchange) are ordinary kernels on the same stream.
void launch_exchange(serfsim* h, const TickParams& p) {
  const u32 t = p.tick, xpar = p.xpar;
  PublishParams pb{};
  pb.world = p.world; pb.rank = p.rank; pb.stamp = p.stamp; pb.xpar = xpar; pb.send_count = h->d_send_count; pb.peer_ctrl = h->d_peer_ctrl;
  pb.row = p.row; pb.gate = p.gate.ctl; pb.sched = h->d_sched; pb.loopback = p.loopback;
  if (!p.fuse_publish) { launch_publish(pb, h->stream); h->last_launches++; }
  DrainParams d{};
  d.n_local = h->count; d.stride = h->stride; d.R = h->R; d.world = p.world; d.rank = p.rank; d.win_cap = h->win_cap; d.stamp = p.stamp; d.n_tiles = h->n_tiles; d.kinds_prev = p.kinds_prev;
  d.win_data = h->d_win_data[xpar]; d.ctrl = h->d_ctrl + xpar * 16; d.inbox_wr = h->d_inbox[t & 1]; d.hot_wr = h->d_hot[t & 1]; d.kinds_cur = p.kinds_cur; d.overflow = h->d_overflow;
  d.byz_on = h->byz_on ? 1u : 0u; d.byz_delta = h->byz_delta; d.shard_size = h->shard_size; d.rec = h->d_rec; d.node_state = h->d_node; d.peer_anomaly = h->d_peer_anomaly;
  d.ue_n = h->ue_table.n; d.ue_inbox_wr = h->ue_table.n ? h->ue->inbox[t & 1].get() : nullptr; d.ue_ltime = h->ue ? h->ue->ltime.get() : nullptr;
  d.my_row = p.row; d.grow = h->d_grow + (size_t)t * ROW_FIELDS; d.gate = p.gate.ctl;
  d.sums = reinterpret_cast<const u64*>(reinterpret_cast<const unsigned char*>(h->d_ctrl.get()) + CTRL_SUMS_OFF) + (size_t)xpar * 8 * CTRL_FIELDS;
  d.sched = h->d_sched; d.sched_rw = h->d_sched; d.host_idle_until = h->d_pin_ctl + 2; d.tick = t; d.sleep_on = p.sleep_on;
  launch_drain(d, h->stream);
  h->last_launches += 1;
  h->xepoch++;
}

// Anti-entropy round on a snapshot of the end-of-tick state (only this node's own records are written); p: as the membership tick left it.
int anti_entropy_round(serfsim* h, TickParams p) {
  const u32 t = p.tick;
  CU(cudaMemcpyAsync(h->d_snap_rec, h->d_rec, h->d_rec.bytes(), cudaMemcpyDeviceToDevice, h->stream));
  CU(cudaMemcpyAsync(h->d_snap_node, h->d_node, h->d_node.bytes(), cudaMemcpyDeviceToDevice, h->stream));
  if (h->ue_table.n) {
    CU(cudaMemcpyAsync(h->ue->snap, h->ue->state, h->ue->state.bytes(), cudaMemcpyDeviceToDevice, h->stream));
    p.ue_table = h->ue_table; p.ue_state = h->ue->state; p.ue_snap = h->ue->snap; p.ue_snap_peer = h->ue->peer_snap;
    p.ue_ltime = h->ue->ltime; p.ue_totals = h->ue->totals;
  }
  if (h->cfg.world_size > 1) {
    // partners may live on other GPUs: their snapshots are read through the peer mappings.  Rounds are rare (every
    // push_pull_interval ticks) and always the first tick of a convergence chunk, so two host barriers are affordable:
    // every rank has taken its snapshot before anyone reads, everyone has read before anyone moves on.
    p.snap_rec_peer = h->d_peer_snap_rec; p.snap_node_peer = h->d_peer_snap_node;
    CU(cudaStreamSynchronize(h->stream));
    h->barrier(h->comm_user);
    if (h->ue_table.n) {
      // A partner in another shard may hold events this shard has never received, so their Lamport times are not in the
      // local table yet (a shard learns them from the first window entry of the event).  The replay needs them: every rank
      // installs the cluster's times before the round.
      u32 lt[MAX_UEVENTS];
      if (int rc = ue_cluster_ltimes(h, lt)) return rc;
      CU(cudaMemcpy(h->ue->ltime, lt, h->ue->ltime.bytes(), cudaMemcpyHostToDevice));
    }
    launch_pushpull(p, h->d_snap_rec, h->d_snap_node, h->cfg.trace != 0, h->stream);
    CU(cudaStreamSynchronize(h->stream));
    h->barrier(h->comm_user);
    // the round changed this rank's row (changed / pending / hash) after the drain kernel summed the rows: redo the sum through
    // the host hook — the host is in the loop here anyway (two barriers), and rounds are rare
    u64 row[ROW_FIELDS];
    CU(cudaMemcpy(row, h->d_trace + (size_t)t * ROW_FIELDS, sizeof(row), cudaMemcpyDeviceToHost));
    h->allreduce(h->comm_user, row, ROW_FIELDS);
    CU(cudaMemcpy(h->d_grow + (size_t)t * ROW_FIELDS, row, sizeof(row), cudaMemcpyHostToDevice));
  } else {
    launch_pushpull(p, h->d_snap_rec, h->d_snap_node, h->cfg.trace != 0, h->stream);
  }
  h->last_launches++;
  return 0;
}

// Launch n ticks on the stream (no synchronisation).
int launch_ticks(serfsim* h, u32 n) {
  if (!h->has_topo) return fail(SERFSIM_E_INVAL, "serfsim_step: no topology set");
  if (h->cfg.world_size > 1 && !h->connected) return fail(SERFSIM_E_COMM, "serfsim_step: world_size > 1 but serfsim_comm_connect was not called");
  int rc = upload_ops(h);
  if (rc) return rc;
  rc = ensure_trace(h, h->tick + n + 1);
  if (rc) return rc;
  if (!h->timing_open) { CU(cudaEventRecord(h->ev0, h->stream)); h->timing_open = true; h->last_launches = 0; h->launch_log.clear(); h->launch_log_first = h->tick; }
  for (u32 i = 0; i < n; ++i) {
    const u32 t = h->tick;
    const u64 launches_before = h->last_launches;
    const OpRange ops = ops_of_tick(h, t);
    for (u32 k = ops.begin; k < ops.end; ++k) {     // ground truth the SWIM probe observes (after this tick's ops)
      const HostOp& o = h->ops[k];
      const int s = slot_of(h, o.node);
      if (s >= 0) { if (o.op == SERFSIM_OP_FAIL) h->up_mask &= ~(1u << s); if (o.op == SERFSIM_OP_REJOIN) h->up_mask |= (1u << s); }
    }
    if (ops.end > ops.begin) { launch_mark_events(h->d_busy, h->d_hot[(t & 1) ^ 1], h->d_ev_node, ops.begin, ops.end, h->first, h->count, h->stream); h->last_launches++; }
    TickParams p = tick_params(h, t, ops);
    h->ever_down |= p.down_mask;
    if (h->tick_timing) {
      if ((rc = grow_events(h->tick_ev, 2 * ((size_t)t + 1)))) return rc;
      CU(cudaEventRecord(h->tick_ev[2 * (size_t)t], h->stream));
    }
    if (h->sw.l2_window && h->l2_window_max) {
      cudaStreamAttrValue av{};
      av.accessPolicyWindow.base_ptr = h->d_inbox[t & 1];
      av.accessPolicyWindow.num_bytes = std::min(h->d_inbox[t & 1].bytes(), h->l2_window_max);
      av.accessPolicyWindow.hitRatio = (float)std::min(1.0, (double)h->l2_persist_max / (double)std::max<size_t>(1, av.accessPolicyWindow.num_bytes));
      av.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
      av.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
      CU(cudaStreamSetAttribute(h->stream, cudaStreamAttributeAccessPolicyWindow, &av));
    }
    if (h->ue_table.n) launch_user_events(h, p);
    launch_membership(h, p);
    if (h->byz_n) launch_injectors(h, p);
    if (h->cfg.world_size > 1) {
      if (h->tick_timing) {
        if ((rc = grow_events(h->mid_ev, (size_t)t + 1))) return rc;
        CU(cudaEventRecord(h->mid_ev[t], h->stream));
      }
      launch_exchange(h, p);
    }
    if (pp_tick(h, t) && (rc = anti_entropy_round(h, p))) return rc;
    if (h->tick_timing) CU(cudaEventRecord(h->tick_ev[2 * (size_t)t + 1], h->stream));
    h->launch_log.push_back((u32)(h->last_launches - launches_before));
    h->tick++;
  }
  CU(cudaGetLastError());
  return 0;
}

int finish_timing(serfsim* h) {
  if (!h->timing_open) return 0;
  CU(cudaEventRecord(h->ev1, h->stream));
  CU(cudaEventSynchronize(h->ev1));
  float ms = 0.f;
  CU(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  h->last_ms = ms; h->timing_open = false; h->launches += h->last_launches;
  return 0;
}

int check_overflow(serfsim* h) {
  if (h->ue_table.n) {
    // Cluster runs need one Lamport time per ring slot: the packed event record derives a slot's ltime from the events in it.
    // (Two tracked events 512·k apart would alias — the quirk itself is kept in ue_handle and pinned by the handler tests.)
    u32 lt[MAX_UEVENTS];
    if (int rc = ue_cluster_ltimes(h, lt)) return rc;
    for (u32 a = 0; a < h->ue_table.n; ++a)
      for (u32 b = a + 1; b < h->ue_table.n; ++b) {
        const bool fa = ((h->ue_injected >> a) & 1u) && h->ue_fire_tick[a] < h->tick, fb = ((h->ue_injected >> b) & 1u) && h->ue_fire_tick[b] < h->tick;
        if (fa && fb && lt[a] % UE_RING == lt[b] % UE_RING && lt[a] != lt[b])
          return fail(SERFSIM_E_INVAL, "user events: two tracked events share a ring slot with different Lamport times (not supported in cluster runs)");
      }
  }
  CU(cudaStreamSynchronize(h->stream));
  const u32 ov = *(volatile u32*)h->pin_overflow;
  if (ov == 1) return fail(SERFSIM_E_OVERFLOW, "a Lamport time or incarnation left the 32-bit device range");
  if (ov == 2) return fail(SERFSIM_E_COMM, "cross-shard window overflow (raise SERFSIM_WIN_FACTOR)");
  if (ov == 4) return fail(SERFSIM_E_INVAL, "single-view check (SERFSIM_SV=2): a view outside the set of views with business had business");
  if (ov) return fail(SERFSIM_E_COMM, "corrupt cross-shard window entry");
  return 0;
}

int pull_rows(serfsim* h) {                     // bring rows [rows.size(), tick) to the host (global sums when sharded)
  const u32 have = (u32)h->rows.size();
  if (have >= h->tick) return 0;
  const u32 n = h->tick - have;
  h->rows.resize(h->tick);
  // sharded runs: the drain kernel of every tick has already summed the ranks' rows on the device (d_grow), no host collective
  const u64* src = h->cfg.world_size > 1 ? h->d_grow : h->d_trace;
  CU(cudaMemcpy(h->rows.data() + have, src + (size_t)have * ROW_FIELDS, (size_t)n * sizeof(serfsim_tick_row_t), cudaMemcpyDeviceToHost));
  return 0;
}

int fire_events(serfsim* h) {
  if (!h->cb) return 0;
  std::vector<u64> out;
  if (int rc = read_summary(h, out)) return rc;
  for (u32 type = 0; type < 3; ++type) {
    std::vector<u32> ids;
    for (u32 s = 0; s < h->R; ++s) {
      if (out[2 + 2 * s] != out[3 + 2 * s]) continue;                 // views still disagree
      const u8 status = (u8)((out[2 + 2 * s] >> 4) & 0xf);
      const u32 ty = status == ST_ALIVE ? SERFSIM_EVENT_JOIN : status == ST_FAILED ? SERFSIM_EVENT_FAILED : SERFSIM_EVENT_LEAVE;
      if (ty == type && h->reported[s] != status) ids.push_back(h->subj[s]);
    }
    if (!ids.empty()) h->cb(h->cb_user, h->tick, type, ids.data(), (u32)ids.size());
  }
  for (u32 s = 0; s < h->R; ++s) if (out[2 + 2 * s] == out[3 + 2 * s]) h->reported[s] = (u8)((out[2 + 2 * s] >> 4) & 0xf);
  return 0;
}

// Watcher masks depend on topology and subjects; the busy bit / hot tiles of the watchers are re-applied after every reset.
int refresh_watchers(serfsim* h) {
  if (!h->has_topo) return 0;
  if (h->watch_dirty) {
    launch_compute_watch(h->d_rowptr, h->d_col, h->d_subj, h->R, h->first, h->count, h->d_watch, h->stream);
    h->watch_dirty = false;
  }
  CU(h->d_hot_static.fill(0, h->stream));
  launch_apply_watch(h->d_watch, h->count, h->d_busy, h->d_hot_static, h->stream);
  CU(cudaGetLastError());
  return 0;
}

int ue_reset(serfsim* h) {                      // bootstrap event state: clock 1, nothing seen, nothing queued
  h->ue_injected = 0;
  if (!h->ue_table.n) return 0;
  launch_ue_init(h->ue->state, h->count, h->stream);
  CU(h->ue->inbox[0].fill(0, h->stream)); CU(h->ue->inbox[1].fill(0, h->stream));
  CU(h->ue->ltime.fill(0, h->stream)); CU(h->ue->totals.fill(0, h->stream));
  CU(cudaGetLastError());
  return 0;
}

int do_reset(serfsim* h, u64 seed) {
  h->cfg.seed = seed; h->tick = 0; h->ops.clear(); h->op_keys.clear(); h->ops_dirty = false; h->rows.clear();
  h->up_mask = (h->R >= 32) ? 0xffffffffu : ((1u << h->R) - 1);
  h->ever_down = 0;
  h->reported.assign(h->R, (u8)ST_ALIVE);
  launch_init_state(h->d_rec, h->d_node, h->count, h->stride, h->R, h->cfg.init_status_ltime, h->cfg.init_clock, h->stream);
  CU(h->d_inbox[0].fill(0, h->stream)); CU(h->d_inbox[1].fill(0, h->stream));
  CU(cudaStreamSynchronize(h->stream));                   // no kernel of an earlier run is still writing the error word
  *(volatile u32*)h->pin_overflow = 0;
  ((volatile u32*)h->pin_ctl)[2] = 0;                     // the scheduler's "sleep until" word (mirrors d_sched, cleared below)
  CU(h->d_busy.fill(0, h->stream)); CU(h->d_qword.fill(0, h->stream));
  CU(h->d_hot[0].fill(0, h->stream)); CU(h->d_hot[1].fill(0, h->stream));
  CU(h->d_tile_due.fill(0xff, h->stream)); CU(h->d_node_due.fill(0xff, h->stream));      // no timer runs
  CU(h->d_carry.fill(0, h->stream));                     // tags restart with the ticks
  CU(h->d_sched.fill(0, h->stream));
  CU(h->d_trace.fill(0, h->stream)); CU(h->d_kinds.fill(0, h->stream)); CU(h->d_view_kinds.fill(0, h->stream)); CU(h->d_grow.fill(0, h->stream));
  CU(h->d_runctl.fill(0, h->stream)); CU(h->d_send_count.fill(0, h->stream));
  { int rc = ue_reset(h); if (rc) return rc; }
  if (h->byz) { CU(h->byz->anomaly.fill(0, h->stream)); CU(h->byz->totals.fill(0, h->stream)); }
  { int rc = refresh_watchers(h); if (rc) return rc; }
  CU(cudaStreamSynchronize(h->stream));
  return 0;
}

// A peer's exported buffer mapped into this process (unmapped when the handle is destroyed).
template <class T>
int ipc_open(serfsim* h, const cudaIpcMemHandle_t& handle, const char* what, T** out) {
  IpcMapping m;
  const cudaError_t e = m.create(handle);
  if (e != cudaSuccess) return fail(SERFSIM_E_COMM, std::string("cudaIpcOpenMemHandle(") + what + "): " + cudaGetErrorString(e));
  *out = (T*)(void*)m;
  h->ipc_opened.push_back(std::move(m));
  return 0;
}

int getter(serfsim* h, u32 slot, int what, void* out, size_t elem) {
  if (!h || !out) return fail(SERFSIM_E_INVAL, "null argument");
  if (what != EXTRACT_CLOCK && what != EXTRACT_CLOCK32 && slot >= h->R) return fail(SERFSIM_E_INVAL, "slot out of range");
  launch_extract(h->d_rec, h->d_node, h->count, h->stride, slot, what, h->d_stage, h->stream);
  CU(cudaMemcpyAsync(out, h->d_stage, (size_t)h->count * elem, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  return 0;
}

}  // namespace

// hooks for wire_codec.cu (the other translation unit behind the C ABI)
namespace sfs {
struct WireView { const uint4* rec; const u32* qword; const u64* node_state; const uint4* ue_state; const u32* subj; u32 n_local, stride, R; cudaStream_t stream; wire::UeWire ue; };
int serfsim_fail(int code, const char* msg) { return fail(code, msg); }
int serfsim_wire_view(const serfsim* h, WireView* out) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  *out = WireView{h->d_rec, h->d_qword, h->d_node, h->ue_table.n ? h->ue->state.get() : nullptr, h->d_subj, h->count, h->stride, h->R, h->stream, h->ue_wire};
  out->ue.ltime = h->ue ? h->ue->ltime.get() : nullptr;
  return 0;
}
}  // namespace sfs

// =====================================================================================
// C ABI
// =====================================================================================
#pragma GCC visibility push(default)
extern "C" {

uint32_t serfsim_abi_version(void) { return SERFSIM_ABI_VERSION; }
const char* serfsim_last_error(void) { return g_err.c_str(); }

void serfsim_default_config(serfsim_config_t* c) {
  if (!c) return;
  memset(c, 0, sizeof(*c));
  c->abi_version = SERFSIM_ABI_VERSION;
  c->n_nodes = 0; c->slots = 1;
  c->fanout = 3;                       // memberlist LAN gossip_nodes
  c->retransmit_mult = 4; c->suspicion_mult = 4; c->suspicion_max_timeout_mult = 6;
  c->probe_interval_ticks = 5;         // 1 s / 200 ms
  c->gossip_interval_ms = 200;
  c->init_status_ltime = 1; c->init_clock = 2;
  c->trace = 0; c->seed = 1; c->device = -1; c->rank = 0; c->world_size = 1;
  c->push_pull_interval_ticks = 0;     // LAN: 30 s = 150 ticks × pushPullScale(n); off unless asked for
  c->reap_interval_ticks = 0;          // options.rs:506: 15 s = 75 ticks; off unless asked for
  c->tombstone_timeout_ticks = 432000; c->reconnect_timeout_ticks = 432000;   // 24 h (options.rs:508-509)
  c->recent_intent_timeout_ticks = 1500;                                     // 5 min (options.rs:515)
}

int serfsim_create(const serfsim_config_t* cfg, serfsim_t** out) {
  if (!cfg || !out) return fail(SERFSIM_E_INVAL, "null argument");
  *out = nullptr;
  if (cfg->abi_version != SERFSIM_ABI_VERSION) return fail(SERFSIM_E_INVAL, "abi_version mismatch");
  if (cfg->n_nodes < 2 || cfg->slots < 1 || cfg->slots > MAX_SLOTS || cfg->fanout < 1 || cfg->fanout > MAX_FANOUT)
    return fail(SERFSIM_E_INVAL, "bad n_nodes / slots (1..16) / fanout (1..8)");
  if (cfg->world_size < 1 || cfg->rank < 0 || cfg->rank >= cfg->world_size) return fail(SERFSIM_E_INVAL, "bad rank / world_size");
  if (cfg->gossip_interval_ms == 0) return fail(SERFSIM_E_INVAL, "gossip_interval_ms must be > 0");
  if (cfg->push_pull_interval_ticks < 0) return fail(SERFSIM_E_INVAL, "push_pull_interval_ticks must be >= 0");
  if (cfg->suspicion_mult >= 2 && cfg->suspicion_mult - 2 > MAX_K) return fail(SERFSIM_E_INVAL, "suspicion_mult too large");
  if (cfg->init_clock >= INIT_LTIME_BOUND) return fail(SERFSIM_E_INVAL, "init_clock must be below LTIME_LIMIT - 16 (0x7FFFFFE0)");
  if (cfg->init_status_ltime >= INIT_LTIME_BOUND) return fail(SERFSIM_E_INVAL, "init_status_ltime must be below LTIME_LIMIT - 16 (0x7FFFFFE0)");
  {
    const u64 limit = retransmit_limit(cfg->retransmit_mult, cfg->n_nodes);
    if (limit == 0 || limit > 255) return fail(SERFSIM_E_INVAL, "retransmit limit (retransmit_mult x digits of n_nodes) must be 1..255");
    const u32 probe = cfg->probe_interval_ticks ? cfg->probe_interval_ticks : 1;
    const char* why = suspicion_table_unrepresentable(cfg->suspicion_mult, cfg->suspicion_max_timeout_mult, probe, cfg->gossip_interval_ms, cfg->n_nodes);
    if (why) return fail(SERFSIM_E_INVAL, why);
    for (u32 t : suspicion_table(cfg->suspicion_mult, cfg->suspicion_max_timeout_mult, probe, cfg->gossip_interval_ms, cfg->n_nodes))
      if (t > TIMEOUT_LIMIT_TICKS) return fail(SERFSIM_E_INVAL, kTimeoutTooLong);      // the double step rounded past the bound
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(SERFSIM_E_NO_DEVICE, "no CUDA device: serfsim has no CPU execution path");
  if (cfg->device >= 0) { if (cfg->device >= ndev) return fail(SERFSIM_E_NO_DEVICE, "device ordinal out of range"); CU(cudaSetDevice(cfg->device)); }
  int dev = 0, major = 0, minor = 0;
  CU(cudaGetDevice(&dev));
  CU(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  CU(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (major != 9 || minor != 0) return fail(SERFSIM_E_NO_DEVICE, "kernels are built for sm_90a only (H100)");

  std::unique_ptr<serfsim> h(new serfsim());
  h->cfg = *cfg; h->N = cfg->n_nodes; h->R = cfg->slots;
  h->shard_size = (h->N + cfg->world_size - 1) / cfg->world_size;
  h->first = std::min<u64>((u64)h->shard_size * cfg->rank, h->N);
  h->count = (u32)std::min<u64>(h->shard_size, (u64)h->N - h->first);
  if (h->count == 0) return fail(SERFSIM_E_INVAL, "empty shard");
  if (h->shard_size >= (1u << 26)) return fail(SERFSIM_E_INVAL, "shard larger than 2^26 nodes");
  h->rules.limit = (u32)retransmit_limit(cfg->retransmit_mult, h->N);      // 1..255: checked above
  auto tab = suspicion_table(cfg->suspicion_mult, cfg->suspicion_max_timeout_mult, cfg->probe_interval_ticks ? cfg->probe_interval_ticks : 1, cfg->gossip_interval_ms, h->N);
  h->rules.k = (u32)tab.size() - 1;
  for (size_t i = 0; i < tab.size(); ++i) h->rules.timeout[i] = tab[i];
  h->subj.resize(h->R);
  for (u32 s = 0; s < h->R; ++s) h->subj[s] = s;

  CU(h->stream.create());
  CU(h->ev0.create()); CU(h->ev1.create());
  h->stride = plane_stride(h->count);
  h->n_tiles = h->stride >> TILE_SHIFT;
  const size_t planes = (size_t)h->R * h->stride;
  CU(h->d_rec.alloc(2 * planes)); CU(h->d_rec.fill(0, h->stream));
  CU(h->d_qword.alloc(planes));
  CU(h->d_inbox[0].alloc(3 * planes)); CU(h->d_inbox[1].alloc(3 * planes));
  CU(h->d_node.alloc(h->stride)); CU(h->d_node.fill(0, h->stream));
  CU(h->d_busy.alloc(h->stride));
  CU(h->d_watch.alloc(h->stride)); CU(h->d_watch.fill(0, h->stream));
  CU(h->d_hot[0].alloc(h->n_tiles)); CU(h->d_hot[1].alloc(h->n_tiles));
  CU(h->d_hot_static.alloc(h->n_tiles)); CU(h->d_hot_static.fill(0, h->stream));
  CU(h->d_tile_due.alloc(h->n_tiles)); CU(h->d_node_due.alloc(h->stride)); CU(h->d_sched.alloc(SCHED_WORDS));
  if (h->R > 1 && cfg->world_size <= 1) CU(h->d_carry.alloc(h->stride));
  CU(h->pin_overflow.create(1)); CU(cudaHostGetDevicePointer(&h->d_overflow, h->pin_overflow, 0));
  CU(h->d_subj.alloc(MAX_SLOTS)); CU(h->d_scratch.alloc(64));
  CU(h->d_stage.alloc(h->count));
  CU(h->d_runctl.alloc(2));
  CU(h->pin_ctl.create(4)); CU(cudaHostGetDevicePointer(&h->d_pin_ctl, h->pin_ctl, 0));
  CU(cudaMemcpy(h->d_subj, h->subj.data(), h->R * 4, cudaMemcpyHostToDevice));
  h->sw = read_switches();
  cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, dev);
  if (h->sms <= 0) h->sms = 132;
  const int ctas_r1 = cfg->world_size > 1 ? tick_ctas_per_sm_r1s() : tick_ctas_per_sm_r1();
  h->ctas_per_sm = h->R > 1 ? tick_ctas_per_sm_rn() : h->sw.minb5 ? 5 : ctas_r1;
  h->grid = tick_grid_size(h->count, h->ctas_per_sm, h->sms, h->sw.gridmul);
  h->grid_sv = tick_grid_size(h->count, ctas_r1, h->sms, h->sw.gridmul);
  {
    // L2 set-aside for persisting (evict_last) lines: the randomly addressed inbox planes live there
    int max_persist = 0, max_window = 0;
    cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, dev);
    cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, dev);
    h->l2_persist_max = (size_t)max_persist; h->l2_window_max = (size_t)max_window;
    if (h->sw.l2_persist && max_persist > 0) cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, (size_t)max_persist);
    if (h->sw.verbose) fprintf(stderr, "serfsim: L2 persisting max %d B, window max %d B, persist %d window %d\n", max_persist, max_window, h->sw.l2_persist, (int)h->sw.l2_window);
  }
  if (cfg->world_size > 1) {
    // receive windows: one segment per peer; expected entries per tick and pair ≈ shard · fanout · R · kinds / world
    if (cfg->world_size > 8) return fail(SERFSIM_E_INVAL, "world_size > 8");
    // … plus what a warp of the tick kernel (TILE threads) can leave unfilled in a peer's window: its reservation ahead and a partial block
    const double pad = (double)std::max(h->grid, h->grid_sv) * (TILE / 32) * (XW_RESERVE_MAX + XW_FLUSH);   // (the single-view kernel of a multi-slot run has the larger grid)
    double cap = (double)h->shard_size * cfg->fanout * h->R * 3.0 * h->sw.win_factor / cfg->world_size + 4096.0 + pad;
    h->win_cap = (u32)std::min(cap, 4.0e9);
    h->win_cap_base = h->win_cap;
    for (int par = 0; par < 2; ++par) {
      CU(h->d_win_data[par].alloc((size_t)cfg->world_size * h->win_cap));
      CU(h->d_win_data[par].fill(0, h->stream));      // windows read as zeros wherever nothing was written
      CU(h->d_peer_data[par].alloc(8));
    }
    CU(h->d_ctrl.alloc(CTRL_BYTES / sizeof(u32))); CU(h->d_ctrl.fill(0, h->stream));
    CU(h->d_send_count.alloc(8));
    CU(h->d_peer_ctrl.alloc(8));
    serfsim::Injectors b; CU(b.anomaly.alloc(h->stride)); CU(b.totals.alloc(4)); h->byz = std::move(b);   // peers' drain kernels raise the flags
    CU(h->d_peer_anomaly.alloc(8));
  }
  if (cfg->push_pull_interval_ticks > 0) {         // push-pull rounds' snapshots (sharded runs export them, so all are allocated here)
    CU(h->d_snap_rec.alloc(h->d_rec.size())); CU(h->d_snap_node.alloc(h->d_node.size()));
    if (cfg->world_size > 1) { CU(h->d_peer_snap_rec.alloc(8)); CU(h->d_peer_snap_node.alloc(8)); }
  }
  if (int rc = ensure_trace(h.get(), 1024)) return rc;
  if (int rc = do_reset(h.get(), cfg->seed)) return rc;
  *out = h.release();
  return 0;
}

void serfsim_destroy(serfsim_t* h) {
  if (!h) return;
  cudaStreamSynchronize(h->stream);
  if (h->sw.xtiming && !h->mid_ev.empty()) {
    double a = 0, b = 0; size_t n = std::min(h->mid_ev.size(), h->tick_ev.size() / 2);
    for (size_t t = 0; t < n; ++t) {
      float x = 0, y = 0;
      if (cudaEventElapsedTime(&x, h->tick_ev[2 * t], h->mid_ev[t]) == cudaSuccess && cudaEventElapsedTime(&y, h->mid_ev[t], h->tick_ev[2 * t + 1]) == cudaSuccess) {
        a += x; b += y;
        if (t >= 12 && t <= 15) fprintf(stderr, "rank %d tick %zu: tick kernel %.1f us, publish+drain %.1f us\n", h->cfg.rank, t, x * 1e3, y * 1e3);
      }
    }
    fprintf(stderr, "rank %d: tick kernels %.3f ms, publish+drain %.3f ms over %zu ticks\n", h->cfg.rank, a, b, n);
  }
  delete h;
}

int serfsim_set_topology_csr(serfsim_t* h, const uint64_t* row_ptr, const uint32_t* col_idx) {
  if (!h || !row_ptr || !col_idx) return fail(SERFSIM_E_INVAL, "null argument");
  if (row_ptr[0] != 0) return fail(SERFSIM_E_INVAL, "row_ptr[0] must be 0");
  const u64 e0 = row_ptr[h->first], e1 = row_ptr[h->first + h->count];
  if (e1 < e0 || e1 - e0 >= 0xffffffffull) return fail(SERFSIM_E_INVAL, "shard has too many edges (u32 offsets)");
  std::vector<u32> rp((size_t)h->stride + 8);
  for (u32 i = 0; i <= h->count; ++i) {
    const u64 r = row_ptr[h->first + i];
    if (r < e0 || (i && r < row_ptr[h->first + i - 1])) return fail(SERFSIM_E_INVAL, "row_ptr not monotone");
    if (i && r - row_ptr[h->first + i - 1] > 65535) return fail(SERFSIM_E_INVAL, "node degree > 65535 (peer draws are 16-bit)");
    rp[i] = (u32)(r - e0);
  }
  const u64 ne = e1 - e0;
  h->udeg = (h->count && ne % h->count == 0) ? (u32)(ne / h->count) : 0u;
  for (u32 i = 0; i <= h->count && h->udeg; ++i) if (rp[i] != (u64)i * h->udeg) h->udeg = 0;
  if (!h->sw.udeg) h->udeg = 0;
  for (size_t i = h->count + 1; i < rp.size(); ++i) rp[i] = (u32)ne;      // padding rows: degree 0
  h->max_tile_edges = 0;
  for (u32 b = 0; b < h->count; b += 256) {
    const u32 lo = rp[b] & ~3u, hi = (rp[std::min<u32>(b + 256, h->count)] + 3u) & ~3u;
    h->max_tile_edges = std::max(h->max_tile_edges, hi - lo);
  }
  for (u64 i = 0; i < ne; ++i) if (col_idx[e0 + i] >= h->N) return fail(SERFSIM_E_INVAL, "col_idx out of range");
  DevArray<u32> d_rowptr, d_col;                  // installed together once both hold the new topology
  CU(d_rowptr.alloc(rp.size()));
  CU(d_col.alloc(ne + 8));
  CU(cudaMemset(d_col, 0, d_col.bytes()));
  CU(cudaMemcpy(d_rowptr, rp.data(), d_rowptr.bytes(), cudaMemcpyHostToDevice));
  if (ne) CU(cudaMemcpy(d_col, col_idx + e0, ne * 4, cudaMemcpyHostToDevice));
  h->d_rowptr = std::move(d_rowptr); h->d_col = std::move(d_col);
  // TMA pipeline (single-slot runs): a stage holds the largest tile's CSR span if that is at most 48 KB
  h->stage_col_bytes = 0;
  {
    const u32 need = std::max<u32>(h->max_tile_edges * 4u, 16u);    // the direct-load kernel is the default (DESIGN §5)
    if (h->sw.tma && h->R == 1 && need <= 48u * 1024u) h->stage_col_bytes = (need + 127u) & ~127u;
  }
  h->grid = tick_grid_size(h->count, h->stage_col_bytes ? 3 : h->ctas_per_sm, h->sms, h->sw.gridmul);
  if (h->sw.verbose) fprintf(stderr, "serfsim: tick kernel = %s (stage_col_bytes %u, grid %d)\n", h->stage_col_bytes ? "tick_kernel_tma" : "tick_kernel", h->stage_col_bytes, h->grid);
  h->has_topo = true;
  h->watch_dirty = true;
  return refresh_watchers(h);
}

int serfsim_set_subjects(serfsim_t* h, const uint32_t* subjects) {
  if (!h || !subjects) return fail(SERFSIM_E_INVAL, "null argument");
  if (h->tick != 0) return fail(SERFSIM_E_INVAL, "subjects can only change at tick 0");
  for (u32 i = 0; i < h->R; ++i) {
    if (subjects[i] >= h->N) return fail(SERFSIM_E_INVAL, "subject id out of range");
    for (u32 j = 0; j < i; ++j) if (subjects[j] == subjects[i]) return fail(SERFSIM_E_INVAL, "subjects must be distinct");
  }
  h->subj.assign(subjects, subjects + h->R);
  CU(cudaMemcpy(h->d_subj, h->subj.data(), h->R * 4, cudaMemcpyHostToDevice));
  h->watch_dirty = true;
  // tick 0 with a clean state: re-derive the watchers' busy bits / hot tiles for the new subjects
  CU(h->d_busy.fill(0, h->stream)); CU(h->d_hot[0].fill(0, h->stream)); CU(h->d_hot[1].fill(0, h->stream));
  return refresh_watchers(h);
}

int serfsim_reset(serfsim_t* h, uint64_t seed) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  return do_reset(h, seed);
}

int serfsim_inject(serfsim_t* h, uint32_t tick, uint32_t op, uint32_t node, uint32_t slot) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  if (tick < h->tick) return fail(SERFSIM_E_INVAL, "cannot schedule an operation in the past");
  if (node >= h->N || op < SERFSIM_OP_JOIN || op > SERFSIM_OP_FORCE_LEAVE_PRUNE) return fail(SERFSIM_E_INVAL, "bad node / op");
  if (op == SERFSIM_OP_USER_EVENT) {
    if (slot >= h->ue_table.n) return fail(SERFSIM_E_INVAL, "user event index out of range (serfsim_set_user_events)");
    if ((h->ue_injected >> slot) & 1u) return fail(SERFSIM_E_INVAL, "a tracked user event can be injected once");
  }
  if (op == SERFSIM_OP_FORCE_LEAVE || op == SERFSIM_OP_FORCE_LEAVE_PRUNE) { if (slot >= h->R) return fail(SERFSIM_E_INVAL, "slot out of range"); }
  else if ((op == SERFSIM_OP_JOIN || op == SERFSIM_OP_LEAVE) && slot_of(h, node) < 0)
    return fail(SERFSIM_E_INVAL, "join/leave origin must be a tracked subject");
  if (!h->op_keys.insert(((u64)tick << 32) | node).second) return fail(SERFSIM_E_INVAL, "one operation per node per tick");
  if (op == SERFSIM_OP_USER_EVENT) { h->ue_injected |= 1u << slot; h->ue_origin[slot] = node; h->ue_fire_tick[slot] = tick; }
  h->ops.push_back(HostOp{tick, op, node, slot, h->op_seq++});
  h->ops_dirty = true;
  return 0;
}

int serfsim_step(serfsim_t* h, uint32_t n_ticks) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  int rc = launch_ticks(h, n_ticks);
  if (rc) return rc;
  rc = finish_timing(h);
  if (rc) return rc;
  rc = check_overflow(h);
  if (rc) return rc;
  return fire_events(h);
}

int serfsim_run_until_converged(serfsim_t* h, uint32_t max_ticks, uint32_t* ticks_out) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  // Ticks are launched in chunks WITHOUT looking at their rows: the first kernel of every tick evaluates the quiescence rule
  // on the previous tick's (global) row on the device and, once the run is over, it and every later kernel return at once
  // (tick_kernel.cuh: Gate).  The host reads two words per chunk; ranks of a sharded run reach the same verdict from the same
  // device-summed rows, so there is no host collective in the loop.  Ticks launched past the first quiescent one never
  // execute: nothing to rewind on the device, the logical clock (and the exchange epoch) is simply set back.
  // Chunks start small and grow (8, 16, 32) — and start small again after every jump over a sleeping stretch: a tick launched into a
  // cluster that has just gone to sleep (or has just finished) still costs its launches (5 – 11 µs: two kernels per tick in multi-slot
  // runs; in sharded runs it even executes), a synchronisation costs less than two of them.  The leave + fail study (877 ticks, ≈ 70 of
  // them busy) launched 382 ticks per run with chunks of up to 128.
  u32 chunk = 8, chunk_max = 32;
  if (h->sw.chunk) chunk = chunk_max = h->sw.chunk;
  const u32 pp = (u32)std::max(0, h->cfg.push_pull_interval_ticks);
  const u32 start = h->tick;
  int rc = 0;
  CU(cudaMemsetAsync(h->d_runctl, 0, 2 * sizeof(u32), h->stream));
  h->pin_ctl[0] = h->pin_ctl[1] = 0;                   // nothing of an earlier call is in flight: every call ends synchronised
  h->gate_on = true; h->gate_first = start;
  struct GateOff { serfsim* h; ~GateOff() { h->gate_on = false; } } gate_off{h};
  auto finish = [&](u32 converged_at, bool converged) -> int {
    if ((rc = finish_timing(h))) return rc;
    if ((rc = check_overflow(h))) return rc;
    if (ticks_out) *ticks_out = converged_at;
    if ((rc = fire_events(h))) return rc;
    return converged ? 0 : 1;
  };
  auto stop_at = [&](u32 t) {                         // tick t is the first quiescent one: later launches did not execute
    const u32 skipped = h->tick - (t + 1);
    if (h->cfg.world_size > 1) h->xepoch -= skipped;   // skipped ticks exchanged nothing
    h->tick = t + 1;
    if (h->rows.size() > h->tick) h->rows.resize(h->tick);
    u64 executed = 0;                                  // kernels of the ticks that did run (launch_log starts at launch_log_first)
    for (u32 k = 0; k < h->launch_log.size() && h->launch_log_first + k <= t; ++k) executed += h->launch_log[k];
    h->last_launches = executed;
  };
  bool probe = false;                                  // the next launch is the single tick whose gate judges the row the jump starts from
  while (h->tick - start < max_ticks) {
    const u32 n = probe ? 1u : std::min(chunk, max_ticks - (h->tick - start));
    if ((rc = launch_ticks(h, n))) return rc;
    CU(cudaStreamSynchronize(h->stream));
    if (h->sw.debug_loop) fprintf(stderr, "loop: launched %u ticks -> tick %u, ctl %u %u until %u probe %d chunk %u\n", n, h->tick, h->pin_ctl[0], h->pin_ctl[1], h->pin_ctl[2], (int)probe, chunk);
    if (*(volatile u32*)h->pin_ctl) {
      const u32 t = ((volatile u32*)h->pin_ctl)[1];
      stop_at(t);
      return finish(t, true);
    }
    if (!probe) chunk = std::min(chunk * 2, chunk_max);
    // The last executed tick proved that nothing can happen before tick `until` (tick_kernel.cu: finish_tick): the ticks up to
    // there — and up to the next host operation — are not even launched; one small kernel writes their rows.  The rows a jump
    // produces equal the row before it, and that one must have been judged "not quiescent" by a gate first: a jump is
    // preceded by one single-tick launch (`probe`).
    const u32 until = ((volatile u32*)h->pin_ctl)[2];
    const bool sleeping = !h->sw.no_jump && until > h->tick && h->tick - start < max_ticks;      // sharded runs: every rank reads the same word
    // … and the probe tick itself must have been an idle one: with a host operation in it (which may well change nothing) its row is a new
    // one that no gate has judged yet — the next launch is another single tick (found by fuzz scenario 16 once the launch chunks ended
    // on the tick before a no-op operation: the run was reported quiescent at the end of the jump instead of at the operation's tick)
    const bool probe_was_idle = !(probe && h->tick > 0 && ops_at(h, h->tick - 1));
    if (sleeping && probe && probe_was_idle) {
      u32 stop = until;
      const u32 nxt = ops_of_tick(h, h->tick).begin;    // the first operation at or after this tick
      if (nxt < h->ops.size()) stop = std::min(stop, h->ops[nxt].tick);
      const u32 n_skip = std::min(stop > h->tick ? stop - h->tick : 0u, max_ticks - (h->tick - start));
      if (n_skip) {
        if ((rc = ensure_trace(h, h->tick + n_skip + 1))) return rc;
        launch_fill_idle_rows(h->d_trace + (size_t)h->tick * 8, h->cfg.world_size > 1 ? h->d_grow + (size_t)h->tick * 8 : nullptr, n_skip, h->d_sched, h->cfg.trace != 0, h->stream);
        h->last_launches++;
        SFS_COUNT(17, n_skip);                           // ticks the host jumped over
        for (u32 k = 0; k < n_skip; ++k) {
          if (h->tick_timing) {
            const u32 t = h->tick + k;
            if ((rc = grow_events(h->tick_ev, 2 * ((size_t)t + 1)))) return rc;
            CU(cudaEventRecord(h->tick_ev[2 * (size_t)t], h->stream)); CU(cudaEventRecord(h->tick_ev[2 * (size_t)t + 1], h->stream));
          }
          h->launch_log.push_back(k == 0 ? 1u : 0u);
        }
        h->tick += n_skip;
        if (!h->sw.chunk) chunk = 8;            // the busy stretch after a sleep is short as a rule
      }
      probe = false;
    } else {
      probe = sleeping;
    }
  }
  // max_ticks reached: the last tick's row has not been judged by any kernel yet — apply the same rule here
  if (h->tick > start) {
    if ((rc = pull_rows(h))) return rc;
    const u32 t = h->tick - 1;
    if (quiescent_row((const u64*)&h->rows[t], t, future_ops(h, t), pp, h->byz_on)) return finish(t, true);
  }
  return finish(h->tick, false);
}

int serfsim_shard_range(serfsim_t* h, uint32_t* first, uint32_t* count) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  if (first) *first = h->first;
  if (count) *count = h->count;
  return 0;
}
int serfsim_member_status(serfsim_t* h, uint32_t slot, uint8_t* out) { return getter(h, slot, EXTRACT_STATUS, out, 1); }
int serfsim_status_ltime(serfsim_t* h, uint32_t slot, uint64_t* out) { return getter(h, slot, EXTRACT_STATUS_LTIME, out, 8); }
int serfsim_lamport_time(serfsim_t* h, uint64_t* out) { return getter(h, 0, EXTRACT_CLOCK, out, 8); }
// compact variants: the device keeps Lamport times in 32 bits (a run that would leave that range fails with SERFSIM_E_OVERFLOW), so
// the same values can cross PCIe at half the size
int serfsim_status_ltime_u32(serfsim_t* h, uint32_t slot, uint32_t* out) { return getter(h, slot, EXTRACT_STATUS_LTIME32, out, 4); }
int serfsim_lamport_time_u32(serfsim_t* h, uint32_t* out) { return getter(h, 0, EXTRACT_CLOCK32, out, 4); }
int serfsim_incarnation(serfsim_t* h, uint32_t slot, uint32_t* out) { return getter(h, slot, EXTRACT_INC, out, 4); }
int serfsim_ml_state(serfsim_t* h, uint32_t slot, uint8_t* out) { return getter(h, slot, EXTRACT_ML, out, 1); }

// The step's result vectors without stalling the launch stream: the three extractions run on the launch stream (in order after
// the ticks), the device→host copies on a second stream.  The caller may start its next step at once; the copies overlap its
// ticks.  Host buffers must stay valid (and should be pinned) until serfsim_results_wait returns.
int serfsim_results_async(serfsim_t* h, uint32_t slot, uint8_t* status, uint32_t* status_ltime, uint32_t* lamport) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  if (slot >= h->R) return fail(SERFSIM_E_INVAL, "slot out of range");
  const size_t n = h->count, n4 = ((n * 4 + 255) / 256) * 256;
  if (!h->rb) {
    serfsim::ReadBack r;
    CU(r.copy_stream.create()); CU(r.extracted.create());
    for (serfsim::ResBuf& b : r.res) { CU(b.d.alloc(2 * n4 + n)); CU(b.copied.create()); }
    h->rb = std::move(r);
  }
  serfsim::ReadBack& rb = *h->rb;
  serfsim::ResBuf& b = rb.res[rb.next++ & 3u];
  if (b.used) CU(cudaStreamWaitEvent(h->stream, b.copied, 0));            // the copy that last read this staging buffer has finished
  if (status_ltime) launch_extract(h->d_rec, h->d_node, h->count, h->stride, slot, EXTRACT_STATUS_LTIME32, b.d, h->stream);
  if (lamport) launch_extract(h->d_rec, h->d_node, h->count, h->stride, slot, EXTRACT_CLOCK32, b.d + n4, h->stream);
  if (status) launch_extract(h->d_rec, h->d_node, h->count, h->stride, slot, EXTRACT_STATUS, b.d + 2 * n4, h->stream);
  CU(cudaEventRecord(rb.extracted, h->stream));
  CU(cudaStreamWaitEvent(rb.copy_stream, rb.extracted, 0));
  if (status_ltime) CU(cudaMemcpyAsync(status_ltime, b.d, n * 4, cudaMemcpyDeviceToHost, rb.copy_stream));
  if (lamport) CU(cudaMemcpyAsync(lamport, b.d + n4, n * 4, cudaMemcpyDeviceToHost, rb.copy_stream));
  if (status) CU(cudaMemcpyAsync(status, b.d + 2 * n4, n, cudaMemcpyDeviceToHost, rb.copy_stream));
  CU(cudaEventRecord(b.copied, rb.copy_stream));
  b.used = true;
  return 0;
}
int serfsim_results_wait(serfsim_t* h) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  if (h->rb) CU(cudaStreamSynchronize(h->rb->copy_stream));
  return 0;
}

int serfsim_records(serfsim_t* h, uint32_t slot, void* out) {
  if (!h || !out) return fail(SERFSIM_E_INVAL, "null argument");
  if (slot >= h->R) return fail(SERFSIM_E_INVAL, "slot out of range");
  DevArray<uint4> tmp;                           // merged image: record | transmit budgets of the queue word
  CU(tmp.alloc(2 * (size_t)h->count));
  launch_compose_records(h->d_rec, h->d_qword, h->count, h->stride, slot, tmp, h->stream);
  CU(cudaMemcpyAsync(out, tmp, tmp.bytes(), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  return 0;
}

int serfsim_tick_trace(serfsim_t* h, uint32_t first_tick, uint32_t n, serfsim_tick_row_t* out) {
  if (!h || !out) return fail(SERFSIM_E_INVAL, "null argument");
  if ((u64)first_tick + n > h->tick) return fail(SERFSIM_E_INVAL, "trace range beyond the executed ticks");
  CU(cudaStreamSynchronize(h->stream));
  int rc = pull_rows(h);
  if (rc) return rc;
  memcpy(out, h->rows.data() + first_tick, (size_t)n * sizeof(serfsim_tick_row_t));
  return 0;
}

int serfsim_state_hash(serfsim_t* h, uint64_t* out) {
  if (!h || !out) return fail(SERFSIM_E_INVAL, "null argument");
  CU(cudaMemsetAsync(h->d_scratch, 0, 4 * 8, h->stream));
  launch_state_hash(h->d_rec, h->d_qword, h->d_node, h->count, h->stride, h->first, h->N, h->R, h->d_scratch, h->stream);
  if (h->ue_table.n) launch_ue_summary(h->ue->state, h->count, h->first, h->N, h->R, h->ue_table.n, h->d_scratch + 1, h->stream);
  u64 parts[4] = {0, 0, 0, 0};
  CU(cudaMemcpyAsync(parts, h->d_scratch, 4 * 8, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  *out = parts[0] + parts[3];                    // records + node words, plus the event records when user events are on
  if (h->cfg.world_size > 1) {
    if (!h->allreduce) return fail(SERFSIM_E_COMM, "world_size > 1: serfsim_comm_set_hooks was not called");
    h->allreduce(h->comm_user, out, 1);
  }
  return 0;
}

int serfsim_stats(serfsim_t* h, serfsim_stats_t* o) {
  if (!h || !o) return fail(SERFSIM_E_INVAL, "null argument");
  memset(o, 0, sizeof(*o));
  CU(cudaStreamSynchronize(h->stream));
  int rc = pull_rows(h);
  if (rc) return rc;
  o->tick = h->tick; o->members = h->N;
  for (size_t i = 0; i < h->rows.size(); ++i) {
    const auto& r = h->rows[i];
    o->packets += r.packets; o->edge_updates += r.edge_updates; o->messages += r.messages; o->changed += r.changed; o->events += r.events;
    if (r.pending || r.edge_updates || r.events) o->last_active_tick = i;
  }
  if (!h->rows.empty()) o->pending = h->rows.back().pending;
  std::vector<u64> out;
  if ((rc = read_summary(h, out))) return rc;
  o->member_time = out[0]; o->intent_queue = out[1];
  for (u32 s = 0; s < h->R; ++s) if (out[2 + 2 * s] != ~0ull && out[2 + 2 * s] != out[3 + 2 * s]) o->disagree_slots++;
  return 0;
}

// ---- byzantine injectors (BASELINE configs[4]; model in byz.cuh) ----
int serfsim_set_byzantine(serfsim_t* h, uint32_t n, const uint32_t* ids, uint32_t delta) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  if (n && !ids) return fail(SERFSIM_E_INVAL, "null ids");
  if (h->tick != 0 || !h->ops.empty()) return fail(SERFSIM_E_INVAL, "serfsim_set_byzantine: call before any operation is scheduled (or after serfsim_reset)");
  if (n && h->cfg.world_size > 1 && h->shard_size >= BYZ_FLAG) return fail(SERFSIM_E_INVAL, "byzantine injectors: shards must hold fewer than 2^25 nodes");
  std::vector<u32> v(ids, ids + n);
  std::sort(v.begin(), v.end());
  for (u32 i = 0; i < n; ++i) if (v[i] >= h->N || (i && v[i] == v[i - 1])) return fail(SERFSIM_E_INVAL, "byzantine ids must be distinct node ids");
  std::vector<u32> mine;                           // every rank is given the global list and keeps the injectors of its shard
  for (u32 id : v) if (id - h->first < h->count) mine.push_back(id);
  DevArray<u32> d_ids;
  if (!mine.empty()) {
    CU(d_ids.alloc(mine.size()));
    CU(cudaMemcpy(d_ids, mine.data(), d_ids.bytes(), cudaMemcpyHostToDevice));
  }
  if (n && !h->byz) { serfsim::Injectors b; CU(b.anomaly.alloc(h->stride)); CU(b.totals.alloc(4)); h->byz = std::move(b); }
  if (h->byz) h->byz->ids = std::move(d_ids);
  h->byz_n = (u32)mine.size(); h->byz_delta = delta; h->byz_on = n != 0;
  if (n) { CU(cudaMemset(h->byz->anomaly, 0, h->byz->anomaly.bytes())); CU(cudaMemset(h->byz->totals, 0, h->byz->totals.bytes())); }
  return 0;
}

int serfsim_anomaly_flags(serfsim_t* h, uint8_t* out) {
  if (!h || !out) return fail(SERFSIM_E_INVAL, "null argument");
  if (!h->byz_on) return fail(SERFSIM_E_INVAL, "no byzantine injectors set (serfsim_set_byzantine)");
  CU(cudaStreamSynchronize(h->stream));
  if (h->cfg.world_size > 1) {                     // peers' drain kernels raise flags in this array: wait until every rank has drained
    if (!h->barrier) return fail(SERFSIM_E_COMM, "world_size > 1: serfsim_comm_set_hooks was not called");
    h->barrier(h->comm_user);
  }
  CU(cudaMemcpy(out, h->byz->anomaly, h->count, cudaMemcpyDeviceToHost));
  return 0;
}

int serfsim_byzantine_stats(serfsim_t* h, serfsim_byz_stats_t* o) {
  if (!h || !o) return fail(SERFSIM_E_INVAL, "null argument");
  if (!h->byz_on) return fail(SERFSIM_E_INVAL, "no byzantine injectors set (serfsim_set_byzantine)");
  u64 t[4] = {0, 0, 0, 0};
  CU(cudaStreamSynchronize(h->stream));
  if (h->cfg.world_size > 1) {
    if (!h->barrier || !h->allreduce) return fail(SERFSIM_E_COMM, "world_size > 1: serfsim_comm_set_hooks was not called");
    h->barrier(h->comm_user);                      // see serfsim_anomaly_flags
  }
  CU(cudaMemcpy(t, h->byz->totals, h->byz->totals.bytes(), cudaMemcpyDeviceToHost));
  std::vector<u8> flags(h->count);
  CU(cudaMemcpy(flags.data(), h->byz->anomaly, h->count, cudaMemcpyDeviceToHost));
  u64 v[3] = {t[0], t[1], 0};
  for (u8 f : flags) v[2] += f ? 1 : 0;
  if (h->cfg.world_size > 1) h->allreduce(h->comm_user, v, 3);
  o->messages = v[0]; o->edge_updates = v[1]; o->flagged = v[2];
  return 0;
}

// ---- user events (SURVEY §8f row 3; rules in uevent.cuh) ----
int serfsim_set_user_events(serfsim_t* h, uint32_t n_events, const uint32_t* content_ids) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  if (n_events > MAX_UEVENTS) return fail(SERFSIM_E_INVAL, "at most SERFSIM_MAX_USER_EVENTS tracked user events");
  if (n_events && !content_ids) return fail(SERFSIM_E_INVAL, "null content ids");
  if (h->tick != 0 || !h->ops.empty()) return fail(SERFSIM_E_INVAL, "serfsim_set_user_events: call before any operation is scheduled (or after serfsim_reset)");
  if (h->cfg.world_size > 1) {
    // every event bit bound for another shard is one window entry: up to fanout · n_events per node and tick on top of the
    // membership entries the windows were sized for.  The windows are exported by serfsim_comm_export, so this must come first.
    const double cap = (double)h->win_cap_base + (double)h->shard_size * h->cfg.fanout * n_events * h->sw.win_factor / h->cfg.world_size;
    const u32 want = (u32)std::min(cap, 4.0e9);
    if (want != h->win_cap) {
      if (h->connected) return fail(SERFSIM_E_INVAL, "serfsim_set_user_events: in sharded runs call it before serfsim_comm_export / serfsim_comm_connect (it resizes the receive windows)");
      for (int par = 0; par < 2; ++par) { CU(h->d_win_data[par].alloc((size_t)h->cfg.world_size * want)); CU(h->d_win_data[par].fill(0, h->stream)); }
      h->win_cap = want;
    }
  }
  if (n_events && !h->ue) {
    const bool pp = h->cfg.push_pull_interval_ticks > 0;
    if (pp && h->connected) return fail(SERFSIM_E_INVAL, "serfsim_set_user_events: in sharded runs with push-pull rounds call it before serfsim_comm_export (the event snapshot is exported)");
    serfsim::UserEvents u;
    CU(u.state.alloc(h->stride)); CU(u.inbox[0].alloc(h->stride)); CU(u.inbox[1].alloc(h->stride));
    CU(u.ltime.alloc(MAX_UEVENTS)); CU(u.totals.alloc(8));
    if (pp) { CU(u.snap.alloc(h->stride)); CU(u.peer_snap.alloc(8)); }
    h->ue = std::move(u);
  }
  h->ue_table = UeTable{};
  h->ue_table.n = n_events;
  h->ue_wire.n = 0;                               // a new event table drops the content of the old one
  for (u32 e = 0; e < n_events; ++e) h->ue_table.content[e] = content_ids[e];
  int rc = ue_reset(h);
  if (rc) return rc;
  CU(cudaStreamSynchronize(h->stream));
  return 0;
}

// The bytes of the tracked events, encoded once into their UserEvents.events entries (wire.cuh) for the batch encoder.
int serfsim_set_user_event_content(serfsim_t* h, uint32_t n, const uint8_t* const* names, const size_t* name_lens, const uint8_t* const* payloads,
                                   const size_t* payload_lens) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  if (!n || n != h->ue_table.n) return fail(SERFSIM_E_INVAL, "serfsim_set_user_event_content: n must equal the n_events of serfsim_set_user_events (> 0)");
  if (!names || !name_lens || !payloads || !payload_lens) return fail(SERFSIM_E_INVAL, "null argument");
  for (u32 e = 0; e < n; ++e) {
    if ((name_lens[e] && !names[e]) || (payload_lens[e] && !payloads[e])) return fail(SERFSIM_E_INVAL, "null argument");
    // Serf::user_event (serf/api.rs:251-282): name + payload within max_user_event_size, then the encoded message with its
    // envelope as well — at the widest Lamport time the device can stamp (5 varint bytes) and cc = false
    if (name_lens[e] > wire::MAX_USER_EVENT_SIZE || payload_lens[e] > wire::MAX_USER_EVENT_SIZE || name_lens[e] + payload_lens[e] > wire::MAX_USER_EVENT_SIZE)
      return fail(SERFSIM_E_INVAL, "user event " + std::to_string(e) + ": name + payload exceed max_user_event_size (512)");
    if (wire::envelope_len(wire::uem_payload_len(0xffffffffull, (u32)name_lens[e], (u32)payload_lens[e], false)) > wire::MAX_USER_EVENT_SIZE)
      return fail(SERFSIM_E_INVAL, "user event " + std::to_string(e) + ": the encoded UserEventMessage exceeds max_user_event_size (512)");
  }
  auto bytes_eq = [&](u32 a, u32 b) {
    return name_lens[a] == name_lens[b] && payload_lens[a] == payload_lens[b] && (!name_lens[a] || !memcmp(names[a], names[b], name_lens[a])) &&
           (!payload_lens[a] || !memcmp(payloads[a], payloads[b], payload_lens[a]));
  };
  for (u32 a = 0; a < n; ++a)
    for (u32 b = a + 1; b < n; ++b) {
      const bool same_id = h->ue_table.content[a] == h->ue_table.content[b], same_bytes = bytes_eq(a, b);
      if (same_id != same_bytes)                     // the device de-duplicates by id, a real node by bytes: they must agree
        return fail(SERFSIM_E_INVAL, "user events " + std::to_string(a) + " and " + std::to_string(b) +
                                     (same_id ? ": equal content ids but different bytes" : ": different content ids but equal bytes"));
    }
  wire::UeWire t{};
  std::vector<u8> buf;
  for (u32 e = 0; e < n; ++e) {
    const u32 nl = (u32)name_lens[e], pl = (u32)payload_lens[e];
    t.off[e] = (u32)buf.size();
    buf.resize(buf.size() + wire::ues_event_entry_len(nl, pl));
    u8* p = buf.data() + t.off[e];
    u32 o = 0;
    p[o++] = wire::UES_EVENT; o += wire::varint_put(p + o, wire::user_event_len(nl, pl));
    t.bytes[e].name_off = t.off[e] + o + (nl ? 1 + wire::varint_len(nl) : 0); t.bytes[e].name_len = nl;
    t.bytes[e].pay_off = t.off[e] + o + (nl ? wire::len_delim_len(nl) : 0) + (pl ? 1 + wire::varint_len(pl) : 0); t.bytes[e].pay_len = pl;
    o += wire::put_user_event(p + o, names[e], nl, payloads[e], pl);
    if (o != wire::ues_event_entry_len(nl, pl)) return fail(SERFSIM_E_INVAL, "wire: internal length mismatch");
  }
  t.off[n] = (u32)buf.size();
  t.n = n;
  if (!h->d_ue_entries) CU(h->d_ue_entries.alloc(wire::UE_TABLE_MAX * wire::UE_ENTRY_MAX));
  CU(cudaStreamSynchronize(h->stream));             // no wire kernel is still reading the old table
  CU(cudaMemcpy(h->d_ue_entries, buf.data(), buf.size(), cudaMemcpyHostToDevice));
  t.entries = h->d_ue_entries;
  h->ue_wire = t;
  return 0;
}

int serfsim_event_time(serfsim_t* h, uint64_t* out) {
  if (!h || !out) return fail(SERFSIM_E_INVAL, "null argument");
  if (!h->ue_table.n) return fail(SERFSIM_E_INVAL, "user events are off (serfsim_set_user_events)");
  launch_ue_extract(h->ue->state, h->count, 0, 0, h->d_stage, h->stream);
  CU(cudaMemcpyAsync(out, h->d_stage, (size_t)h->count * 8, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  return 0;
}

int serfsim_user_event_seen(serfsim_t* h, uint32_t event, uint8_t* out) {
  if (!h || !out) return fail(SERFSIM_E_INVAL, "null argument");
  if (event >= h->ue_table.n) return fail(SERFSIM_E_INVAL, "user event index out of range");
  launch_ue_extract(h->ue->state, h->count, 1, event, h->d_stage, h->stream);
  CU(cudaMemcpyAsync(out, h->d_stage, (size_t)h->count, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  return 0;
}

int serfsim_user_event_ltime(serfsim_t* h, uint32_t event, uint64_t* ltime) {
  if (!h || !ltime) return fail(SERFSIM_E_INVAL, "null argument");
  if (event >= h->ue_table.n) return fail(SERFSIM_E_INVAL, "user event index out of range");
  if (h->cfg.world_size > 1 && !h->allreduce) return fail(SERFSIM_E_COMM, "world_size > 1: serfsim_comm_set_hooks was not called");
  u32 lt[MAX_UEVENTS];
  CU(cudaStreamSynchronize(h->stream));
  if (int rc = ue_cluster_ltimes(h, lt)) return rc;
  *ltime = lt[event];
  return 0;
}

int serfsim_user_event_records(serfsim_t* h, void* out) {
  if (!h || !out) return fail(SERFSIM_E_INVAL, "null argument");
  if (!h->ue_table.n) return fail(SERFSIM_E_INVAL, "user events are off (serfsim_set_user_events)");
  CU(cudaStreamSynchronize(h->stream));
  CU(cudaMemcpy(out, h->ue->state, (size_t)h->count * 16, cudaMemcpyDeviceToHost));
  return 0;
}

int serfsim_user_event_stats(serfsim_t* h, serfsim_uevent_stats_t* o) {
  if (!h || !o) return fail(SERFSIM_E_INVAL, "null argument");
  memset(o, 0, sizeof(*o));
  if (!h->ue_table.n) return fail(SERFSIM_E_INVAL, "user events are off (serfsim_set_user_events)");
  u64 tot[8] = {0}, sum[3] = {0, 0, 0};
  CU(cudaMemsetAsync(h->d_scratch, 0, 3 * 8, h->stream));
  launch_ue_summary(h->ue->state, h->count, h->first, h->N, h->R, h->ue_table.n, h->d_scratch, h->stream);
  CU(cudaMemcpyAsync(sum, h->d_scratch, 3 * 8, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaMemcpyAsync(tot, h->ue->totals, h->ue->totals.bytes(), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  u64 v[6] = {tot[0], tot[1], tot[2], tot[3], tot[4], sum[0]};
  if (h->cfg.world_size > 1) {                      // counters are sums over shards; event_time (a maximum) stays shard-local
    if (!h->allreduce) return fail(SERFSIM_E_COMM, "world_size > 1: serfsim_comm_set_hooks was not called");
    h->allreduce(h->comm_user, v, 6);
  }
  o->messages = v[0]; o->edge_updates = v[1]; o->delivered = v[2]; o->duplicates = v[3]; o->too_old = v[4];
  o->event_queue = v[5]; o->event_time = sum[1];
  return 0;
}

int serfsim_set_event_cb(serfsim_t* h, serfsim_event_cb cb, void* user) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  h->cb = cb; h->cb_user = user;
  return 0;
}

int serfsim_last_step_device_ms(serfsim_t* h, double* ms, uint64_t* kernel_launches) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  if (ms) *ms = h->last_ms;
  if (kernel_launches) *kernel_launches = h->last_launches;
  return 0;
}

int serfsim_set_tick_timing(serfsim_t* h, int enabled) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  h->tick_timing = enabled != 0;
  return 0;
}

int serfsim_tick_times(serfsim_t* h, uint32_t first_tick, uint32_t n, float* ms_out) {
  if (!h || !ms_out) return fail(SERFSIM_E_INVAL, "null argument");
  if (((size_t)first_tick + n) * 2 > h->tick_ev.size()) return fail(SERFSIM_E_INVAL, "tick timing was not enabled for that range");
  CU(cudaStreamSynchronize(h->stream));
  for (u32 i = 0; i < n; ++i) CU(cudaEventElapsedTime(ms_out + i, h->tick_ev[2 * ((size_t)first_tick + i)], h->tick_ev[2 * ((size_t)first_tick + i) + 1]));
  return 0;
}
int serfsim_tick_view_kinds(serfsim_t* h, uint32_t first_tick, uint32_t n, uint32_t* out) {
  if (!h || !out) return fail(SERFSIM_E_INVAL, "null argument");
  if ((size_t)first_tick + n > h->tick) return fail(SERFSIM_E_INVAL, "ticks not run yet");
  if (!n) return 0;
  std::vector<u32> rows((size_t)n * h->R * 4);
  CU(cudaMemcpyAsync(rows.data(), h->d_view_kinds + ((size_t)first_tick + 1) * h->R * 4, rows.size() * sizeof(u32), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  for (size_t i = 0; i < (size_t)n * h->R; ++i)
    for (u32 k = 0; k < 3; ++k) out[i * 3 + k] = rows[i * 4 + k];
  return 0;
}

// ---- multi-GPU: CUDA IPC windows ----------------------------------------------------------
struct comm_blob { cudaIpcMemHandle_t data[2]; cudaIpcMemHandle_t ctrl; cudaIpcMemHandle_t snap_rec, snap_node, anomaly, ue_snap; u32 win_cap; u32 rank; u32 has_snap; u32 has_ue_snap; unsigned char dev_uuid[16]; };

size_t serfsim_comm_blob_size(void) { return sizeof(comm_blob); }

int serfsim_comm_export(serfsim_t* h, void* blob) {
  if (!h || !blob) return fail(SERFSIM_E_INVAL, "null argument");
  if (h->cfg.world_size < 2) return fail(SERFSIM_E_INVAL, "world_size == 1: nothing to export");
  comm_blob b{};
  for (int par = 0; par < 2; ++par) CU(cudaIpcGetMemHandle(&b.data[par], h->d_win_data[par]));
  CU(cudaIpcGetMemHandle(&b.ctrl, h->d_ctrl));
  CU(cudaIpcGetMemHandle(&b.anomaly, h->byz->anomaly));
  if (h->ue && h->ue->snap) { CU(cudaIpcGetMemHandle(&b.ue_snap, h->ue->snap)); b.has_ue_snap = 1; }
  b.win_cap = h->win_cap; b.rank = (u32)h->cfg.rank;
#ifndef SERFSIM_EMU
  { int dev = 0; cudaDeviceProp pr{}; CU(cudaGetDevice(&dev)); CU(cudaGetDeviceProperties(&pr, dev)); memcpy(b.dev_uuid, pr.uuid.bytes, 16); }
#endif
  if (h->d_snap_rec) {                              // push-pull rounds are on: partners on other GPUs read these
    CU(cudaIpcGetMemHandle(&b.snap_rec, h->d_snap_rec)); CU(cudaIpcGetMemHandle(&b.snap_node, h->d_snap_node));
    b.has_snap = 1;
  }
  memcpy(blob, &b, sizeof(b));
  return 0;
}

int serfsim_comm_connect(serfsim_t* h, const void* blobs) {
  if (!h || !blobs) return fail(SERFSIM_E_INVAL, "null argument");
  const int W = h->cfg.world_size;
  if (W < 2) return fail(SERFSIM_E_INVAL, "world_size == 1");
  if (!h->barrier || !h->allreduce) return fail(SERFSIM_E_COMM, "serfsim_comm_set_hooks must be called first");
  const comm_blob* bs = (const comm_blob*)blobs;
  std::vector<u32*> pc(8, nullptr);
  std::vector<std::vector<u64*>> pd(2, std::vector<u64*>(8, nullptr));
  std::vector<const uint4*> psr(8, nullptr);
  std::vector<const u64*> psn(8, nullptr);
  std::vector<u8*> pan(8, nullptr);
  std::vector<const uint4*> pus(8, nullptr);
  const uint4* ue_snap = h->ue ? h->ue->snap.get() : nullptr;
  for (int r = 0; r < W; ++r) {
    if (bs[r].rank != (u32)r || bs[r].win_cap != h->win_cap) return fail(SERFSIM_E_COMM, "blob order / window size mismatch");
#ifndef SERFSIM_EMU
    // one rank per GPU: the drain kernel spins on its peers' flags, and a peer that shares this GPU may never get an SM to raise them
    for (int r2 = 0; r2 < r; ++r2) if (!h->loopback && memcmp(bs[r].dev_uuid, bs[r2].dev_uuid, 16) == 0) return fail(SERFSIM_E_COMM, "two ranks share one GPU (one process per GPU is required)");
#endif
    if ((bs[r].has_snap != 0) != (h->d_snap_rec != nullptr)) return fail(SERFSIM_E_COMM, "push_pull_interval_ticks differs between ranks");
    if (r == h->cfg.rank) { pd[0][r] = h->d_win_data[0]; pd[1][r] = h->d_win_data[1]; pc[r] = h->d_ctrl; psr[r] = h->d_snap_rec; psn[r] = h->d_snap_node; pan[r] = h->byz->anomaly; pus[r] = ue_snap; continue; }
    if ((bs[r].has_ue_snap != 0) != (ue_snap != nullptr)) return fail(SERFSIM_E_COMM, "user events / push-pull configuration differs between ranks");
    int rc = bs[r].has_ue_snap ? ipc_open(h, bs[r].ue_snap, "event snapshot", &pus[r]) : 0;
    if (!rc) rc = ipc_open(h, bs[r].anomaly, "flags", &pan[r]);
    if (!rc && bs[r].has_snap) rc = ipc_open(h, bs[r].snap_rec, "snapshot", &psr[r]);
    if (!rc && bs[r].has_snap) rc = ipc_open(h, bs[r].snap_node, "snapshot", &psn[r]);
    for (int par = 0; par < 2 && !rc; ++par) rc = ipc_open(h, bs[r].data[par], "window", &pd[par][r]);
    if (!rc) rc = ipc_open(h, bs[r].ctrl, "ctrl", &pc[r]);
    if (rc) return rc;
  }
  for (int par = 0; par < 2; ++par) CU(cudaMemcpy(h->d_peer_data[par], pd[par].data(), h->d_peer_data[par].bytes(), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(h->d_peer_ctrl, pc.data(), h->d_peer_ctrl.bytes(), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(h->d_peer_anomaly, pan.data(), h->d_peer_anomaly.bytes(), cudaMemcpyHostToDevice));
  if (ue_snap) CU(cudaMemcpy(h->ue->peer_snap, pus.data(), h->ue->peer_snap.bytes(), cudaMemcpyHostToDevice));
  if (h->d_snap_rec) {
    CU(cudaMemcpy(h->d_peer_snap_rec, psr.data(), h->d_peer_snap_rec.bytes(), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(h->d_peer_snap_node, psn.data(), h->d_peer_snap_node.bytes(), cudaMemcpyHostToDevice));
  }
  h->barrier(h->comm_user);          // every rank has mapped every window before the first tick writes into one
  h->connected = true;
  return 0;
}

int serfsim_comm_loopback(serfsim_t* h) {
  if (!h) return fail(SERFSIM_E_INVAL, "null handle");
  const int W = h->cfg.world_size;
  if (W < 2) return fail(SERFSIM_E_INVAL, "world_size == 1");
  if (h->cfg.rank != 0) return fail(SERFSIM_E_INVAL, "loopback: create the handle as rank 0");
  if (h->cfg.push_pull_interval_ticks > 0 || h->byz_on || h->ue_table.n) return fail(SERFSIM_E_INVAL, "loopback profiles the membership path only");
  // entries for shard s are written at win_data[s][rank·win_cap + g]: with rank 0 the window of "peer" s is my own segment s
  std::vector<u32*> pc(8, nullptr);
  std::vector<std::vector<u64*>> pd(2, std::vector<u64*>(8, nullptr));
  std::vector<u8*> pan(8, nullptr);
  for (int r = 0; r < W; ++r) {
    pc[r] = h->d_ctrl; pan[r] = h->byz->anomaly;
    for (int par = 0; par < 2; ++par) pd[par][r] = h->d_win_data[par] + (size_t)r * h->win_cap;
  }
  for (int par = 0; par < 2; ++par) CU(cudaMemcpy(h->d_peer_data[par], pd[par].data(), h->d_peer_data[par].bytes(), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(h->d_peer_ctrl, pc.data(), h->d_peer_ctrl.bytes(), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(h->d_peer_anomaly, pan.data(), h->d_peer_anomaly.bytes(), cudaMemcpyHostToDevice));
  h->barrier = [](void*) {};
  h->allreduce = [](void*, uint64_t*, uint32_t) {};
  h->connected = true; h->loopback = true;
  return 0;
}

int serfsim_comm_set_hooks(serfsim_t* h, serfsim_barrier_fn barrier, serfsim_allreduce_u64_fn allreduce, void* user) {
  if (!h || !barrier || !allreduce) return fail(SERFSIM_E_INVAL, "null argument");
  h->barrier = barrier; h->allreduce = allreduce; h->comm_user = user;
  return 0;
}

}  // extern "C"
#pragma GCC visibility pop
