/*
 * serfsim.h — C ABI of the H100 gossip-dissemination simulator (drop-in boundary).
 *
 * This is the seam a serf-core `Transport`/`Delegate` shim binds to (Rust `extern "C"` /
 * cudarc-style FFI, see INTEGRATION.md).  Every entry point names the reference
 * interface it replaces; paths are relative to the reference tree
 * (al8n/serf @ b291e49), `serf-core/src/...`.
 *
 * Conventions
 *   - plain pointers + sizes only; no C++ / torch types cross this boundary;
 *   - every function returns 0 on success or a negative SERFSIM_E_* code;
 *     serfsim_last_error() returns a thread-local, NUL-terminated description;
 *   - one host thread drives a handle; event callbacks fire on that thread between ticks
 *     (the reference's delegate methods may be called concurrently,
 *     `delegate.rs:12-14`; here the batch replaces the concurrency);
 *   - host buffers are caller-owned; the library copies in/out (device memory, streams
 *     and the NVLink exchange are internal);
 *   - Lamport times are u64 at this boundary (`types/clock.rs:14`); the device keeps
 *     them as u32 and every call fails with SERFSIM_E_OVERFLOW instead of wrapping.
 *
 * The only backend is CUDA (sm_90a).  There is no CPU fallback: serfsim_create fails
 * with SERFSIM_E_NO_DEVICE when no usable GPU is present.
 */
#ifndef SERFSIM_H
#define SERFSIM_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SERFSIM_ABI_VERSION 4u

/* ---- error codes ------------------------------------------------------------------ */
#define SERFSIM_OK            0
#define SERFSIM_E_INVAL      (-1)   /* bad argument / bad state                          */
#define SERFSIM_E_NO_DEVICE  (-2)   /* no CUDA device / kernels not loadable             */
#define SERFSIM_E_CUDA       (-3)   /* CUDA runtime error other than an allocation failure (text in serfsim_last_error) */
#define SERFSIM_E_NOMEM      (-4)   /* a device, pinned host, stream or event allocation failed (cudaErrorMemoryAllocation) */
#define SERFSIM_E_OVERFLOW   (-5)   /* a Lamport time / incarnation left the u32 device range */
#define SERFSIM_E_COMM       (-6)   /* multi-GPU exchange setup failed                   */

/* ---- MemberStatus — `types/member.rs:54-58` (u8 codes are identical) ---------------- */
#define SERFSIM_STATUS_NONE     0u
#define SERFSIM_STATUS_ALIVE    1u
#define SERFSIM_STATUS_LEAVING  2u
#define SERFSIM_STATUS_LEFT     3u
#define SERFSIM_STATUS_FAILED   4u

/* ---- memberlist node state of a view (external crate memberlist-core 0.8.1,
 *      `proto::State`; restated, see DESIGN.md "SWIM half") --------------------------- */
#define SERFSIM_ML_ALIVE    0u
#define SERFSIM_ML_SUSPECT  1u
#define SERFSIM_ML_DEAD     2u
#define SERFSIM_ML_LEFT     3u

/* ---- MessageType tags carried by intents — `types/message.rs:17-18` ----------------- */
#define SERFSIM_MSG_LEAVE  1u
#define SERFSIM_MSG_JOIN   2u

/* ---- MemberEventType — `event.rs:325-328` (Join, Leave, Failed, Update, Reap) -------- */
#define SERFSIM_EVENT_JOIN    0u
#define SERFSIM_EVENT_LEAVE   1u
#define SERFSIM_EVENT_FAILED  2u
#define SERFSIM_EVENT_UPDATE  3u
#define SERFSIM_EVENT_REAP    4u

/* ---- host-injected operations (what a real node's API call does at its origin) ------- */
#define SERFSIM_OP_JOIN         1u  /* Serf::join → broadcast_join       `serf/api.rs:339-342`, `serf/base.rs:381-397` */
#define SERFSIM_OP_LEAVE        2u  /* Serf::leave                        `serf/api.rs:422-499`                          */
#define SERFSIM_OP_FORCE_LEAVE  3u  /* Serf::remove_failed_node           `serf/base.rs:454-480`                         */
#define SERFSIM_OP_FAIL         4u  /* process crash: node stops sending/receiving (fault injection, cf. MessageDropper `serf/delegate.rs:42-45`) */
#define SERFSIM_OP_REJOIN       5u  /* crashed node returns: memberlist alive(inc+1) + Serf::join                        */
#define SERFSIM_OP_USER_EVENT   6u  /* Serf::user_event                   `serf/api.rs:241-299`; `slot` = tracked user event */
#define SERFSIM_OP_FORCE_LEAVE_PRUNE 7u /* Serf::remove_failed_node_prune `serf/api.rs:513`, `serf/base.rs:454-480` with LeaveMessage.prune
                                           (`types/leave.rs:39-44`): receivers erase the member (handle_prune, `serf/base.rs:1628-1653`) */

#define SERFSIM_MAX_USER_EVENTS 8u

/* ---- configuration: serf `Options` (`options.rs:495-530`) + the memberlist LAN knobs it
 *      embeds (`options.rs:521`), expressed in gossip ticks ----------------------------- */
typedef struct serfsim_config {
  uint32_t abi_version;               /* = SERFSIM_ABI_VERSION                                       */
  uint32_t n_nodes;                   /* N virtual members, dense ids 0..N-1                         */
  uint32_t slots;                     /* R tracked subjects; every node holds a view of each (1..16) */
  uint32_t fanout;                    /* memberlist gossip_nodes (1..8), LAN default 3               */
  uint32_t retransmit_mult;           /* memberlist retransmit_mult, LAN default 4; the limit retransmit_mult x
                                         ceil(log10(n_nodes + 1)), in 64 bits, must be 1..255       */
  uint32_t suspicion_mult;            /* LAN default 4; 0..9 (k = suspicion_mult - 2 <= 7 confirmations) */
  uint32_t suspicion_max_timeout_mult;/* LAN default 6                                               */
  uint32_t probe_interval_ticks;      /* probe_interval / gossip_interval (LAN 1 s / 200 ms = 5); 0 = no probing */
  uint32_t gossip_interval_ms;        /* wall-clock length of one tick (LAN 200); only scales the suspicion table.
                                         The suspicion timeouts' ms arithmetic must fit in int64 and every timeout
                                         must be at most 2^30 ticks (DESIGN.md §2 rule 10)            */
  uint32_t init_status_ltime;         /* bootstrap MemberState.status_time of every view (default 1); < 0x7FFFFFE0 */
  uint32_t init_clock;                /* bootstrap LamportClock of every node (default 2); < 0x7FFFFFE0
                                         (16 below the device's Lamport limit 0x7FFFFFF0)            */
  uint32_t trace;                     /* 1: fill the per-tick state hash (parity runs); 0: skip it   */
  uint64_t seed;                      /* keys the counter RNG (Philox4x32-10)                        */
  int32_t  device;                    /* CUDA ordinal (-1 = current)                                 */
  int32_t  rank;                      /* shard index of this process (0 when world_size == 1)        */
  int32_t  world_size;                /* number of shards (one process per GPU)                      */
  int32_t  push_pull_interval_ticks;  /* memberlist push_pull_interval in ticks (LAN 30 s = 150, times pushPullScale(n)); 0 = no anti-entropy rounds */
  /* Reaper — `serf/base.rs:483-610`, defaults `options.rs:506-515` (reap 15 s = 75 ticks, timeouts 24 h, intents 5 min = 1500 ticks) */
  uint32_t reap_interval_ticks;       /* 0 = the reaper never runs                                                         */
  uint32_t tombstone_timeout_ticks;   /* Left members older than this are erased from the view (Options.tombstone_timeout) */
  uint32_t reconnect_timeout_ticks;   /* Failed members older than this are erased (Options.reconnect_timeout)             */
  uint32_t recent_intent_timeout_ticks; /* buffered intents older than this are dropped (Options.recent_intent_timeout)    */
} serfsim_config_t;

/* ---- Stats — mirrors `serf/api.rs:588-602` (members/failed/left/member_time/intent_queue)
 *      plus the simulator's dissemination counters ------------------------------------ */
typedef struct serfsim_stats {
  uint64_t tick;             /* ticks executed so far                                            */
  uint64_t packets;          /* sender→target deliveries (one UDP packet in the reference)       */
  uint64_t edge_updates;     /* (packet, slot) pairs carrying ≥1 entry: the headline unit        */
  uint64_t messages;         /* individual entries delivered (leave + join + memberlist)         */
  uint64_t changed;          /* merges that changed the destination record ("dirty writes")      */
  uint64_t events;           /* host operations applied                                          */
  uint64_t pending;          /* views still holding queued transmits / timers after last tick    */
  uint64_t last_active_tick; /* last tick that delivered or held anything (convergence marker)   */
  uint64_t members;          /* Stats.members: N                                                 */
  uint64_t member_time;      /* Stats.member_time: max LamportClock over nodes                   */
  uint64_t intent_queue;     /* Stats.intent_queue: queued serf intents over all nodes           */
  uint64_t disagree_slots;   /* slots whose (status, status_time, incarnation, ml) differ among up nodes */
} serfsim_stats_t;

/* One row per executed tick: the convergence trace that must be bit-identical to the CPU
 * event loop (oracle).  `hash` is 0 unless config.trace = 1. */
typedef struct serfsim_tick_row {
  uint64_t packets, edge_updates, messages, changed, pending, events, suspects, hash;
} serfsim_tick_row_t;

/* User-event dissemination counters — Stats.event_time / Stats.event_queue of `serf/api.rs:588-602`
 * plus delivery counters.  Deliveries are also part of the tick rows (edge_updates, messages, changed, pending). */
typedef struct serfsim_uevent_stats {
  uint64_t messages;      /* event messages sent (one per event per target)                                  */
  uint64_t edge_updates;  /* sender→target pairs that carried ≥ 1 event message                               */
  uint64_t delivered;     /* events handed to the application: handle_user_event → true, `serf/base.rs:829-836` */
  uint64_t duplicates;    /* (node, tick, event) arrivals dropped as already seen, `serf/base.rs:801-806`      */
  uint64_t too_old;       /* arrivals outside the event_buffer_size window, `serf/base.rs:771-781`             */
  uint64_t event_queue;   /* Stats.event_queue: event broadcasts still queued, over all nodes                  */
  uint64_t event_time;    /* Stats.event_time: max event LamportClock over nodes                               */
} serfsim_uevent_stats_t;

/* Byzantine stale-record injectors (BASELINE configs[4]).  No reference semantics exist: serf ignores stale intents
 * silently (`serf/base.rs:1346-1348, 1464-1466`); the model is defined by this repository's oracle (DESIGN.md §8). */
typedef struct serfsim_byz_stats {
  uint64_t messages;      /* stale entries injected (one serf + one memberlist entry per peer and subject) */
  uint64_t edge_updates;  /* injected (peer, subject) pairs — NOT part of the tick rows' edge_updates       */
  uint64_t flagged;       /* injectors whose anomaly flag is set                                            */
} serfsim_byz_stats_t;

typedef struct serfsim serfsim_t;   /* opaque; owned by the caller; freed by serfsim_destroy */

/* Batched EventDelegate (`serf/delegate.rs:557-582` notify_join/leave/update → MemberEvent
 * `event.rs:263-293`): called on the driving thread after a step with the ids of the
 * SUBJECTS whose globally agreed status changed.  `type` is SERFSIM_EVENT_*. */
typedef void (*serfsim_event_cb)(void* user, uint32_t tick, uint32_t type,
                                 const uint32_t* ids, uint32_t n);

/* ---- lifecycle — replaces Serf::new / Memberlist::with_delegate (`serf/base.rs:62-344`) */
uint32_t    serfsim_abi_version(void);
void        serfsim_default_config(serfsim_config_t* cfg);            /* memberlist LAN profile, `options.rs:521` */
int         serfsim_create(const serfsim_config_t* cfg, serfsim_t** out);
void        serfsim_destroy(serfsim_t* h);
const char* serfsim_last_error(void);

/* Gossip topology (who a node may pick as gossip/probe peer): CSR over global ids, copied.
 * Every process passes the FULL graph; each keeps the rows of its shard.  Replaces the
 * member list kRandomNodes draws from (memberlist `gossip_nodes`, SURVEY §8c). */
int serfsim_set_topology_csr(serfsim_t* h, const uint64_t* row_ptr /*[N+1]*/, const uint32_t* col_idx /*[row_ptr[N]]*/);

/* Tracked subjects: slot s holds every node's view of member subjects[s] (default: s). */
int serfsim_set_subjects(serfsim_t* h, const uint32_t* subjects /*[slots]*/);

/* Back to the bootstrap state (all members known Alive, clocks = init_clock), tick 0,
 * schedule cleared.  Topology and subjects are kept. */
int serfsim_reset(serfsim_t* h, uint64_t seed);

/* Schedule a host operation at `tick` (≥ current tick).  `node` is the origin; `slot`
 * selects the subject for FORCE_LEAVE (ignored otherwise; JOIN/LEAVE/REJOIN require the
 * origin to be a tracked subject).  == Serf::join / leave / remove_failed_node. */
int serfsim_inject(serfsim_t* h, uint32_t tick, uint32_t op, uint32_t node, uint32_t slot);

/* THE HOT PATH: n_ticks × (receive/state-merge → local ops → timers/probe → gossip send).
 * Replaces, for all N nodes at once: SerfDelegate::notify_message (`serf/delegate.rs:157-315`),
 * handle_node_{join,leave}_intent / handle_node_{join,leave} (`serf/base.rs:1206-1572`),
 * SerfDelegate::broadcast_messages + the TransmitLimitedQueue (`serf/delegate.rs:317-384`,
 * `serf/base.rs:179-190`), LamportClock::witness (`types/clock.rs:155-172`) and memberlist's
 * probe/suspect/dead state machine. */
int serfsim_step(serfsim_t* h, uint32_t n_ticks);

/* Step until no transmit, timer, in-flight message or scheduled operation remains, or
 * max_ticks elapse.  *ticks_out = index of the first quiescent tick (the convergence step
 * count); returns 1 (not an error) when max_ticks was hit first. */
int serfsim_run_until_converged(serfsim_t* h, uint32_t max_ticks, uint32_t* ticks_out);

/* ---- outputs (global order under sharding: rank r fills only its id range unless
 *      world_size == 1; see serfsim_shard_range) -------------------------------------- */
int serfsim_shard_range(serfsim_t* h, uint32_t* first, uint32_t* count);
int serfsim_member_status(serfsim_t* h, uint32_t slot, uint8_t*  out /*[count]*/);  /* Serf::members → Member.status, `serf/api.rs:136-146` */
int serfsim_status_ltime (serfsim_t* h, uint32_t slot, uint64_t* out /*[count]*/);  /* MemberState.status_time, `types/member.rs:23`         */
int serfsim_lamport_time (serfsim_t* h, uint64_t* out /*[count]*/);                 /* LamportClock::time, `types/clock.rs:142`              */
/* The same two vectors at half the size: the device keeps Lamport times in 32 bits (a run that would leave that range fails with
 * SERFSIM_E_OVERFLOW instead of wrapping), so a caller that reads them every step can take them as u32 and widen lazily. */
int serfsim_status_ltime_u32(serfsim_t* h, uint32_t slot, uint32_t* out /*[count]*/);
int serfsim_lamport_time_u32(serfsim_t* h, uint32_t* out /*[count]*/);
/* The same three vectors without stalling the caller (any pointer may be NULL): the extraction is ordered after the ticks on the
 * library's launch stream, the device→host copies run on a second stream and overlap whatever the caller does next (e.g. the
 * ticks of its next study).  The buffers (pinned, ideally) must stay valid until serfsim_results_wait returns. */
int serfsim_results_async(serfsim_t* h, uint32_t slot, uint8_t* status /*[count]*/, uint32_t* status_ltime /*[count]*/, uint32_t* lamport /*[count]*/);
int serfsim_results_wait (serfsim_t* h);
int serfsim_incarnation  (serfsim_t* h, uint32_t slot, uint32_t* out /*[count]*/);  /* memberlist incarnation of the subject as seen         */
int serfsim_ml_state     (serfsim_t* h, uint32_t slot, uint8_t*  out /*[count]*/);  /* SERFSIM_ML_*                                          */
int serfsim_records      (serfsim_t* h, uint32_t slot, void* out /*[count][32]*/);  /* raw 32-byte member records (layout: DESIGN.md)        */
int serfsim_stats        (serfsim_t* h, serfsim_stats_t* out);                       /* Serf::stats, `serf/api.rs:150-183`                    */
int serfsim_tick_trace   (serfsim_t* h, uint32_t first_tick, uint32_t n, serfsim_tick_row_t* out);
int serfsim_state_hash   (serfsim_t* h, uint64_t* out);                              /* hash of all records + clocks, any time                */
int serfsim_set_event_cb (serfsim_t* h, serfsim_event_cb cb, void* user);

/* ---- user events (`Serf::user_event` `serf/api.rs:241-299`, `handle_user_event` `serf/base.rs:750-837`,
 *      re-broadcast `serf/delegate.rs:219-221, 293-300`) ------------------------------------------------
 * Declare the tracked user events: content_ids[e] identifies (name, payload) — two events with equal ids
 * are equal for the receiver's de-duplication.  Event e is fired with
 * serfsim_inject(tick, SERFSIM_OP_USER_EVENT, origin, e), once; its Lamport time is the origin's event
 * clock at that tick.  Call before scheduling operations; n_events = 0 switches user events off.
 * Works sharded (an event crossing shards is one 8-byte window entry carrying its Lamport time; call this BEFORE
 * serfsim_comm_export, it resizes the receive windows; counters of
 * serfsim_user_event_stats are global sums, event_time is the local shard's maximum).  With push-pull rounds on,
 * a round also witnesses the partner's event clock and replays its event ring (`serf/delegate.rs:469-474, 539-552`).
 * Cluster runs need one Lamport time per ring slot: two tracked events 512·k apart fail the run with SERFSIM_E_INVAL
 * (the slot-reuse quirk of handle_user_event is kept in the rules and pinned at handler level). */
int serfsim_set_user_events(serfsim_t* h, uint32_t n_events, const uint32_t* content_ids /*[n_events]*/);
int serfsim_event_time       (serfsim_t* h, uint64_t* out /*[count]*/);                  /* event_clock.time() per node, `serf.rs:139`              */
int serfsim_user_event_seen  (serfsim_t* h, uint32_t event, uint8_t* out /*[count]*/);   /* 1: the node delivered the event to its EventSubscriber */
int serfsim_user_event_ltime (serfsim_t* h, uint32_t event, uint64_t* ltime);            /* UserEventMessage.ltime stamped by the origin (0: not fired yet) */
int serfsim_user_event_records(serfsim_t* h, void* out /*[count][16]*/);                 /* raw 16-byte event records (layout: DESIGN.md)          */
int serfsim_user_event_stats (serfsim_t* h, serfsim_uevent_stats_t* out);

/* ---- byzantine stale-record injectors (BASELINE configs[4]) --------------------------------------------
 * ids[] re-inject, every tick, a copy of their own view aged by `delta` (status_time − delta, incarnation − delta,
 * saturating) to that tick's gossip peers.  anomaly[u] = 1 once a receiver that was up held a view newer than
 * u's injected entry by ≥ delta.  Call before scheduling operations; n = 0 switches injectors off.  With
 * injectors on, serfsim_run_until_converged stops at the first tick with no honest traffic, nothing pending
 * and nothing merged.  Works sharded: every rank passes the GLOBAL id list and keeps the injectors of its shard; an
 * entry bound for another shard is judged by that shard against its own record and the flag is raised in the
 * sender's shard over NVLink.  With push-pull rounds on, the verdict of a tick is taken before that tick's round. */
/* In sharded runs the three calls below and serfsim_user_event_stats / serfsim_user_event_ltime are COLLECTIVE: every rank
 * makes the same calls in the same order (they use the barrier / all-reduce hooks of serfsim_comm_set_hooks). */
int serfsim_set_byzantine  (serfsim_t* h, uint32_t n, const uint32_t* ids /*[n]*/, uint32_t delta);
int serfsim_anomaly_flags  (serfsim_t* h, uint8_t* out /*[count]*/);
int serfsim_byzantine_stats(serfsim_t* h, serfsim_byz_stats_t* out);

/* ---- measurement hooks (bench.py): device time of the tick kernels inside the last
 *      serfsim_step / run_until_converged call, measured with CUDA events on the launch
 *      stream, and the number of kernel launches issued by that call ------------------- */
int serfsim_last_step_device_ms(serfsim_t* h, double* ms, uint64_t* kernel_launches);
/* Optional per-tick device timing (one CUDA event pair per tick, profiling runs only): enable,
 * step, then read the duration in milliseconds of ticks [first_tick, first_tick + n). */
int serfsim_set_tick_timing(serfsim_t* h, int enabled);
int serfsim_tick_times(serfsim_t* h, uint32_t first_tick, uint32_t n, float* ms_out);
/* Messages (leave, join, memberlist entries) each tracked subject's view sent in ticks [first_tick, first_tick + n), as counted by
 * the per-view passes of unsharded multi-slot runs; ticks that ran no passes (host operations, reaper rounds, trace mode, single-slot
 * and sharded runs) read as zero.  out: [n][slots][3]. */
int serfsim_tick_view_kinds(serfsim_t* h, uint32_t first_tick, uint32_t n, uint32_t* out);

/* ---- multi-GPU (one process per GPU; ids sharded by contiguous range) ---------------- */
/* Size of the opaque blob a rank publishes to its peers, and the exchange itself: every
 * rank calls _comm_export, the host side all-gathers the blobs (torch.distributed / MPI /
 * anything), then every rank calls _comm_connect with all blobs in rank order.  The blobs
 * carry CUDA IPC handles of the rank's receive windows; cross-shard gossip payloads are
 * written straight into the peer's window over NVLink by the tick kernel. */
size_t serfsim_comm_blob_size(void);
int    serfsim_comm_export (serfsim_t* h, void* blob);
int    serfsim_comm_connect(serfsim_t* h, const void* blobs /*[world_size][blob_size]*/);
/* Collective hooks the host must provide when world_size > 1 (a barrier and a u64 sum all-reduce across ranks,
 * e.g. torch.distributed / NCCL).  They are NOT on the per-tick data path (that is device-side: peer-window stores,
 * release/acquire flags): the barrier runs once in serfsim_comm_connect, the all-reduce whenever the host looks at
 * trace rows or the state hash (once per convergence-check chunk).  Every rank must make the same sequence of calls.
 * In sharded runs serfsim_stats reports member_time / intent_queue / disagree_slots for the local shard only. */
typedef void (*serfsim_barrier_fn)(void* user);
typedef void (*serfsim_allreduce_u64_fn)(void* user, uint64_t* buf, uint32_t n);
int    serfsim_comm_set_hooks(serfsim_t* h, serfsim_barrier_fn barrier, serfsim_allreduce_u64_fn allreduce, void* user);
/* PROFILING AID (tools/loopback_profile.py): a handle created with world_size = W exchanges with ITSELF — every "peer window"
 * is a segment of its own receive window, so the cross-shard entries of its ticks come back as deliveries into its own shard.
 * One GPU then carries exactly the per-GPU work of a W-rank run (the sharded tick kernel with (W-1)/W of its sends staged and
 * stored into windows, the publish kernel, the drain kernel folding W-1 windows), which makes that path measurable and
 * profilable with ncu on a single GPU.  The simulation results of such a handle are meaningless.  No hooks are needed. */
int    serfsim_comm_loopback(serfsim_t* h);

/* ---- wire codec (SURVEY §8f row 4): serf's TLV encoding of the messages of this path ----------------------------------
 * Join / Leave / PushPull exactly as `types/join.rs:107-158`, `types/leave.rs:121-195`, `types/push_pull.rs:319-450` and the
 * envelope of `types/message.rs:397-428, 507-692` lay them out, ids being u64 (`JoinMessageU64` .. of `types/tests.rs:49-62`).
 * The primitives those files import from the external crate memberlist_core::proto (tag byte, varint, wire types) are restated
 * in serf_b200/csrc/wire.cuh and are UNPINNED at byte level: the crate is not in the reference tree and the tree holds no golden
 * bytes, only the round-trip property (`types/tests.rs:8-25`), which tests/test_wire.py restates. */
#define SERFSIM_WIRE_LEAVE     1u  /* MessageType tags, `types/message.rs:17-19` */
#define SERFSIM_WIRE_JOIN      2u
#define SERFSIM_WIRE_PUSH_PULL 3u
typedef struct { uint32_t type /* SERFSIM_WIRE_JOIN | _LEAVE */, prune /* LeaveMessage.prune */; uint64_t ltime, id; } serfsim_wire_intent_t;
typedef struct {
  uint64_t ltime, event_ltime, query_ltime;         /* `types/push_pull.rs:24-80` */
  uint32_t n_status, n_left;                         /* encode: entries; decode: in = capacity of the arrays, out = entries */
  uint32_t n_events_skipped, pad;                    /* decode: `events` entries present in the message (skipped: not on this path) */
  uint64_t* status_ids; uint64_t* status_ltimes;     /* status_ltimes: IndexMap<Id, LamportTime> in insertion order */
  uint64_t* left_ids;                                /* left_members: IndexSet<Id> */
} serfsim_wire_push_pull_t;
size_t serfsim_wire_encoded_len_intent(const serfsim_wire_intent_t* m);                   /* encoded_message_len, `types/message.rs:484-491` */
int serfsim_wire_encode_intent(const serfsim_wire_intent_t* m, uint8_t* buf, size_t cap, size_t* len);         /* encode_message; *len = needed size even on failure */
int serfsim_wire_encode_push_pull(const serfsim_wire_push_pull_t* m, uint8_t* buf, size_t cap, size_t* len);
int serfsim_wire_message_type(const uint8_t* buf, size_t len, uint32_t* type);            /* decode_message's dispatch, `types/message.rs:507-692` */
int serfsim_wire_decode_intent(const uint8_t* buf, size_t len, serfsim_wire_intent_t* out);
int serfsim_wire_decode_push_pull(const uint8_t* buf, size_t len, serfsim_wire_push_pull_t* out);
/* SerfDelegate::local_state (`serf/delegate.rs:386-425`) of EVERY node of the shard, encoded on the device: message i occupies
 * out[offsets[i] .. offsets[i + 1]).  offsets has count + 1 entries and is always filled; if out is NULL or cap < *total the call
 * fails after setting *total.  A virtual node's member table holds the tracked subjects it knows. */
int serfsim_wire_local_state_batch(serfsim_t* h, uint8_t* out, size_t cap, uint64_t* offsets, size_t* total);
/* The inverse batch on the device: n concatenated push-pull messages → per message the Lamport clock and up to `cap`
 * (id, status_time) entries (arrays [n][cap]) with their count.  Offsets: offsets has n + 1 entries; message i is
 * buf[offsets[i] .. offsets[i + 1]); buf holds at least offsets[n] bytes (they are copied to the device).  Offsets that
 * decrease fail the call with SERFSIM_E_INVAL before anything runs, naming the first bad index.  A malformed message fails
 * the call, naming the lowest such index; a message with more than 16 (MAX_SLOTS) left_members entries counts as one. */
int serfsim_wire_decode_batch(serfsim_t* h, const uint8_t* buf, const uint64_t* offsets, uint32_t n, uint32_t cap,
                              uint64_t* ltime, uint64_t* ids, uint64_t* status_ltimes, uint32_t* n_status);

/* ---- user events on the wire: UserEventMessage (`types/user_event/message.rs`, message type 4), UserEvents / UserEvent
 *      (`types/user_event/user_events.rs`, `types/user_event.rs`) and the `events` field of PushPull (`types/push_pull.rs:455-587`,
 *      one entry per occupied ring slot, in ring-index order).  Decoders return pointers INTO the caller's buffer (no copy);
 *      an empty name or payload decodes as (NULL, 0). ------------------------------------------------------------------------- */
#define SERFSIM_WIRE_USER_EVENT 4u  /* `types/message.rs:20` */
typedef struct {                                     /* UserEventMessage */
  uint64_t ltime;
  const uint8_t* name; size_t name_len;              /* the event name (UTF-8 on a real node; not checked here) */
  const uint8_t* payload; size_t payload_len;
  uint32_t cc, pad;                                  /* "can coalesce" */
} serfsim_wire_user_event_t;
typedef struct { const uint8_t* name; size_t name_len; const uint8_t* payload; size_t payload_len; } serfsim_wire_event_t;   /* UserEvent */
typedef struct { uint64_t ltime; uint32_t n_events, pad; serfsim_wire_event_t* events; } serfsim_wire_user_events_t;         /* UserEvents: one ring slot */
int serfsim_wire_encode_user_event(const serfsim_wire_user_event_t* m, uint8_t* buf, size_t cap, size_t* len);   /* with the envelope; *len = needed size even on failure */
int serfsim_wire_decode_user_event(const uint8_t* buf, size_t len, serfsim_wire_user_event_t* out);
/* PushPull with its ring.  Encode: m as serfsim_wire_encode_push_pull, plus n_ring ring entries written between event_ltime and
 * query_ltime.  Decode: *n_ring / *n_events are in: the capacities of `ring` and of the event pool `events`, out: the entries
 * used (SERFSIM_E_INVAL on a shortfall); ring[k].events points into `events`; out->n_events_skipped is 0. */
int serfsim_wire_encode_push_pull_events(const serfsim_wire_push_pull_t* m, const serfsim_wire_user_events_t* ring, uint32_t n_ring,
                                         uint8_t* buf, size_t cap, size_t* len);
int serfsim_wire_decode_push_pull_events(const uint8_t* buf, size_t len, serfsim_wire_push_pull_t* out, serfsim_wire_user_events_t* ring,
                                         uint32_t* n_ring, serfsim_wire_event_t* events, uint32_t* n_events);
/* The bytes of the tracked user events (the simulator itself knows only content ids): name and payload of event e, as a real
 * node's Serf::user_event(name, payload, cc) would carry them.  Call after serfsim_set_user_events with the same n; the table
 * is kept across serfsim_reset and dropped by the next serfsim_set_user_events.  Rejected (SERFSIM_E_INVAL) when name + payload
 * exceeds max_user_event_size (512, `options.rs:528`), when the encoded UserEventMessage with its envelope would exceed 512
 * bytes (`serf/api.rs:251-282`; checked with a 5-byte Lamport time, the widest the device stamps, and cc = false), or when
 * two events have equal content ids but different bytes or different ids but equal bytes.  Once set, every push-pull message
 * of serfsim_wire_local_state_batch / _range carries the node's event ring; without it the output is as before. */
int serfsim_set_user_event_content(serfsim_t* h, uint32_t n, const uint8_t* const* names, const size_t* name_lens,
                                   const uint8_t* const* payloads, const size_t* payload_lens);
/* serfsim_wire_local_state_batch over the shard-local nodes [first, first + count): message i (node first + i) occupies
 * out[offsets[i] .. offsets[i + 1]), offsets[0] = 0.  The whole-shard batch is this range over every local node, byte for
 * byte.  A node's message can reach a few KB with a content table, so large shards are encoded in chunks. */
int serfsim_wire_local_state_range(serfsim_t* h, uint32_t first, uint32_t count, uint8_t* out, size_t cap, uint64_t* offsets, size_t* total);
/* The rings of n concatenated push-pull messages back to the simulator's form, on the device: per message its event clock
 * (event_ltime), the mask of tracked events its ring holds (bit e: a UserEvent with e's name and payload in an entry whose
 * ltime is e's Lamport time; tracked events with equal content and ltime resolve to the lowest index) and the number of
 * events that match no tracked event.  Needs a content table.  Offsets as for serfsim_wire_decode_batch: n + 1 non-decreasing
 * entries, buf holding at least offsets[n] bytes; decreasing offsets fail the call with SERFSIM_E_INVAL before anything
 * runs.  A malformed message fails the call, naming the lowest such index. */
int serfsim_wire_decode_events_batch(serfsim_t* h, const uint8_t* buf, const uint64_t* offsets, uint32_t n,
                                     uint64_t* event_ltime, uint32_t* seen, uint32_t* n_unmatched);

#ifdef __cplusplus
}
#endif
#endif /* SERFSIM_H */
