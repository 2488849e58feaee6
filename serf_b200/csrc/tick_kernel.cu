// tick_kernel.cu — the fused gossip tick for sm_90a.
//
// One launch = one gossip tick of every virtual node of this shard:
//   Phase R  receive: fold the reduced inbox of the previous tick into the node's views
//            (SerfDelegate::notify_message → handle_node_{join,leave}_intent, serf/delegate.rs:157-315,
//             serf/base.rs:1338-1373, 1442-1572; LamportClock::witness, types/clock.rs:155-172;
//             memberlist alive/suspect/dead merge [external]);
//   Phase E  host operations scheduled for this tick (Serf::join/leave/remove_failed_node, serf/api.rs);
//   Phase T  suspicion-timer expiry and the SWIM probe [external];
//   Phase S  gossip: pick `fanout` distinct peers with the counter RNG and reduce every queued
//            entry into their inbox with RED.MAX (SerfDelegate::broadcast_messages + the
//            TransmitLimitedQueue budget, serf/delegate.rs:317-384, serf/base.rs:179-190).
// Sends of tick t land in inbox parity t&1 and are consumed by Phase R of tick t+1, so a launch
// never reads what it writes: bulk-synchronous, order-independent, bit-reproducible.
//
// Memory behaviour (HBM-bound integer work, no tensor cores): one thread per node; a node's 32-byte record is one DRAM
// sector, read as two back-to-back 128-bit loads (a warp covers 1 KB contiguous) and, if changed, written as two; node
// word, queue word, busy byte and inbox words are coalesced streams with an evict_first / no-L1-allocate policy; the row
// offsets and the four neighbour gathers (evict_first, allocated in L1) stay inside the node's own 64-byte CSR row; the sends are 32-bit RED.MAX to random peers with
// an evict_last policy — the inbox planes are the only randomly addressed data and are sized to stay L2-resident.
// Tiles (256 nodes) nobody delivered to and that hold no pending work are skipped outright in sparse ticks.
// A TMA variant (tick_kernel_tma) stages whole tiles through cp.async.bulk + mbarrier; the multi-GPU variant stages
// cross-shard entries in shared memory and stores them into the peer GPU's window over NVLink.
#include <cstdlib>

#include "tick_kernel.cuh"
#include "byz.cuh"

namespace sfs {

namespace {

constexpr int BLOCK = 256;
#ifndef SFS_MB_R1
// Resident CTAs per SM, i.e. the register cap of each kernel.  Spilled registers go through the LSU the kernels are bound by,
// so the caps are the fastest ones of a sweep on the H100 (DESIGN §5): at 4 CTAs / 64 registers the single-slot kernel
// spills 120–316 B per thread on sm_90a, at 2 CTAs / 128 registers the multi-slot kernel 390–640 B.
#define SFS_MB_R1 3                         // single-slot kernels (80 registers per thread)
#endif
#ifndef SFS_MB_R1S
#define SFS_MB_R1S SFS_MB_R1                // … of the sharded single-slot kernel (its send path needs more registers)
#endif
#ifndef SFS_MB_RN
#define SFS_MB_RN 1                         // multi-slot kernels (up to 255 registers per thread; ptxas uses about 200)
#endif
constexpr u32 MAX_TILES_PER_CTA = 1024;
static_assert(TILE == BLOCK, "tile = block");

// ---- cache-policy plumbing -------------------------------------------------------------------
// The only randomly addressed data of a tick are the inbox planes the sends reduce into (RED.MAX,
// 4 B at a random node).  They are kept L2-resident with an evict_last policy; everything that is
// streamed exactly once per tick (records, node state, the inbox parity being consumed) goes
// through evict_first / no-L1-allocate so it does not push the inbox out of the 50 MB L2.
#ifndef SERFSIM_EMU
__device__ __forceinline__ u64 policy_evict_first() { u64 p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ u64 policy_evict_last() { u64 p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p; }

// sm_90 has no 256-bit LDG/STG: a record is two 128-bit accesses to the two halves of the same 32-byte sector, issued
// back to back so that both are in flight together (the sector crosses DRAM once; the second half is served by L2).
__device__ __forceinline__ Words ld_rec256(const uint4* ptr, u64 pol) {
  Words r;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%8], %9;\n\t"
               "ld.global.L1::no_allocate.L2::cache_hint.v4.u32 {%4,%5,%6,%7}, [%8+16], %9;"
               : "=r"(r.w[0]), "=r"(r.w[1]), "=r"(r.w[2]), "=r"(r.w[3]), "=r"(r.w[4]), "=r"(r.w[5]), "=r"(r.w[6]), "=r"(r.w[7])
               : "l"(ptr), "l"(pol));
  return r;
}
__device__ __forceinline__ void st_rec256(uint4* ptr, const Words& r, u64 pol) {
  asm volatile("st.global.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %9;\n\t"
               "st.global.L2::cache_hint.v4.u32 [%0+16], {%5,%6,%7,%8}, %9;"
               :: "l"(ptr), "r"(r.w[0]), "r"(r.w[1]), "r"(r.w[2]), "r"(r.w[3]), "r"(r.w[4]), "r"(r.w[5]), "r"(r.w[6]), "r"(r.w[7]), "l"(pol) : "memory");
}
__device__ __forceinline__ u64 ld_u64_stream(const u64* ptr, u64 pol) {
  u64 v; asm volatile("ld.global.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(ptr), "l"(pol)); return v;
}
__device__ __forceinline__ u32 ld_u32_stream(const u32* ptr, u64 pol) {
  u32 v; asm volatile("ld.global.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(ptr), "l"(pol)); return v;
}
__device__ __forceinline__ void st_u32_stream(u32* ptr, u32 v, u64 pol) {
  asm volatile("st.global.L2::cache_hint.u32 [%0], %1, %2;" :: "l"(ptr), "r"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_u64_stream(u64* ptr, u64 v, u64 pol) {
  asm volatile("st.global.L2::cache_hint.u64 [%0], %1, %2;" :: "l"(ptr), "l"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void red_max_resident(u32* ptr, u32 v, u64 pol) {   // RED.MAX, result unused, line kept in L2
  asm volatile("red.relaxed.gpu.global.max.L2::cache_hint.u32 [%0], %1, %2;" :: "l"(ptr), "r"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ u32 peek_inbox(const u32* ptr, u64 pol) {   // a word of the plane being reduced into (any value it held during the launch)
  u32 v; asm volatile("ld.global.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(ptr), "l"(pol)); return v;
}
__device__ __forceinline__ u32 ld_u8_stream(const u8* ptr, u64 pol) {
  u32 v; asm volatile("ld.global.L1::no_allocate.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(v) : "l"(ptr), "l"(pol)); return v;
}
__device__ __forceinline__ u32 ld_u16_stream(const u16* ptr, u64 pol) {
  u16 v; asm volatile("ld.global.L1::no_allocate.L2::cache_hint.u16 %0, [%1], %2;" : "=h"(v) : "l"(ptr), "l"(pol)); return v;
}
__device__ __forceinline__ void st_u8_stream(u8* ptr, u32 v, u64 pol) {
  asm volatile("st.global.L2::cache_hint.u8 [%0], %1, %2;" :: "l"(ptr), "r"(v), "l"(pol) : "memory");
}
// A gather from the read-only topology (no write to it during a launch: not volatile, the compiler may schedule it freely), allocated
// in L1: the picks of a node fall into its two CSR sectors, its two row offsets into one, and the later ones hit L1.
__device__ __forceinline__ u32 ld_topo(const u32* ptr, u64 pol) {
  u32 v; asm("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(ptr), "l"(pol)); return v;
}
__device__ __forceinline__ void st_release_sys(u32* ptr, u32 v) { asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(ptr), "r"(v) : "memory"); }
__device__ __forceinline__ u32 ld_acquire_sys(const u32* ptr) { u32 f; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(f) : "l"(ptr) : "memory"); return f; }
#else   // SERFSIM_EMU: the same accessors as plain C++ (tests/emu compiles this file for the host; cache hints have no meaning there)
inline u64 policy_evict_first() { return 0; }
inline u64 policy_evict_last() { return 0; }
// byte counters of the host build (probes 8..14): what the accessors of one run ISSUE, by class — an accounting aid for
// layout experiments (tools/emu_traffic.py), not a DRAM model
inline Words ld_rec256(const uint4* ptr, u64) { emu::probes[8] += 32; Words r; const u32* q = reinterpret_cast<const u32*>(ptr); for (int i = 0; i < 8; ++i) r.w[i] = q[i]; return r; }
inline void st_rec256(uint4* ptr, const Words& r, u64) { emu::probes[9] += 32; u32* q = reinterpret_cast<u32*>(ptr); for (int i = 0; i < 8; ++i) q[i] = r.w[i]; }
inline u64 ld_u64_stream(const u64* ptr, u64) { emu::probes[10] += 8; return *ptr; }
inline u32 ld_u32_stream(const u32* ptr, u64) { emu::probes[11] += 4; return *ptr; }
inline void st_u32_stream(u32* ptr, u32 v, u64) { emu::probes[12] += 4; *ptr = v; }
inline void st_u64_stream(u64* ptr, u64 v, u64) { emu::probes[13] += 8; *ptr = v; }
inline void red_max_resident(u32* ptr, u32 v, u64) { emu::probes[14] += 4; if (v > *ptr) *ptr = v; }
inline u32 peek_inbox(const u32* ptr, u64) { emu::probes[11] += 4; return *ptr; }
inline void st_release_sys(u32* ptr, u32 v) { __atomic_store_n(ptr, v, __ATOMIC_RELEASE); }     // peers are other threads of the test process
inline u32 ld_acquire_sys(const u32* ptr) {                 // polled in a loop by the drain kernel: be polite to the peer threads, and never hang a test run
  static thread_local const u32* last = nullptr;
  static thread_local unsigned long spins = 0;
  if (ptr != last) { last = ptr; spins = 0; }
  if (++spins > 64) emu::polite_wait(spins);
  return __atomic_load_n(ptr, __ATOMIC_ACQUIRE);
}
#endif

// ---- the other per-node planes of a tick, one accessor each with its L2 policy.  Saturated ticks stream them, sparse ticks touch
// them at a few nodes: either way nothing reads them again in the launch, and evict_first keeps them from pushing the inbox planes
// the sends reduce into out of L2 (tools/ubench/pass_mix.cu, DESIGN §5).  Atomics on them (node_due's RED.MIN) keep the default. ----
#ifndef SERFSIM_EMU
__device__ __forceinline__ u32 gather_col(const u32* ptr, u64 pol) { return ld_topo(ptr, pol); }          // CSR neighbour ids
__device__ __forceinline__ u32 ld_row_ptr(const u32* ptr, u64 pol) { return ld_topo(ptr, pol); }          // CSR row offsets (non-uniform degree)
__device__ __forceinline__ u32 ld_qword(const u32* ptr, u64 pol) { return ld_u32_stream(ptr, pol); }      // queue words
__device__ __forceinline__ void st_qword(u32* ptr, u32 v, u64 pol) { st_u32_stream(ptr, v, pol); }
__device__ __forceinline__ u32 ld_busy(const u8* ptr, u64 pol) { return ld_u8_stream(ptr, pol); }        // busy bytes
__device__ __forceinline__ void st_busy(u8* ptr, u32 v, u64 pol) { st_u8_stream(ptr, v, pol); }
__device__ __forceinline__ u32 ld_carry(const u32* ptr, u64 pol) { return ld_u32_stream(ptr, pol); }      // carry words of the passes
__device__ __forceinline__ void st_carry(u32* ptr, u32 v, u64 pol) { st_u32_stream(ptr, v, pol); }
__device__ __forceinline__ u32 ld_node_due(const u32* ptr, u64 pol) { return ld_u32_stream(ptr, pol); }   // a node's own earliest deadline
__device__ __forceinline__ void st_node_due(u32* ptr, u32 v, u64 pol) { st_u32_stream(ptr, v, pol); }
__device__ __forceinline__ u32 ld_watch(const u16* ptr, u64 pol) { return ld_u16_stream(ptr, pol); }     // watcher masks
#else
inline u32 gather_col(const u32* ptr, u64) { return *ptr; }
inline u32 ld_row_ptr(const u32* ptr, u64) { return *ptr; }
inline u32 ld_qword(const u32* ptr, u64) { return *ptr; }
inline void st_qword(u32* ptr, u32 v, u64) { *ptr = v; }
inline u32 ld_busy(const u8* ptr, u64) { return *ptr; }
inline void st_busy(u8* ptr, u32 v, u64) { *ptr = (u8)v; }
inline u32 ld_carry(const u32* ptr, u64) { return *ptr; }
inline void st_carry(u32* ptr, u32 v, u64) { *ptr = v; }
inline u32 ld_node_due(const u32* ptr, u64) { return *ptr; }
inline void st_node_due(u32* ptr, u32 v, u64) { *ptr = v; }
inline u32 ld_watch(const u16* ptr, u64) { return *ptr; }
#endif

#ifndef SERFSIM_EMU
// ---- TMA (bulk async copy) + mbarrier plumbing: stages a whole 256-node tile into shared memory ----
__device__ __forceinline__ u32 smem_u32(const void* p) { return (u32)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(u64* bar, u32 count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(u64* bar, u32 bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(u64* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void mbar_wait(u64* bar, u32 parity) {
  u32 ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// global → shared bulk copy (UBLKCP); completion is signalled on `bar` as transaction bytes
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, u32 bytes, u64* bar, u64 pol) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
}
#endif

// Shared-memory image of one tile (single-slot runs): everything the 256 nodes of the tile read this tick.
constexpr u32 ST_REC = 0, ST_NODE = 8192, ST_INL = 10240, ST_INJ = 11264, ST_INM = 12288, ST_RP = 13312, ST_COL = 14400;
constexpr u32 RP_BYTES = 1040;             // 260 row offsets (257 needed, rounded to 16 B)
struct StageView {
  const Words* rec; const u64* node; const u32* inL; const u32* inJ; const u32* inM; const u32* rowptr; const u32* col;
  u32 col_base;                            // first CSR element held in `col`
  bool col_staged;                         // false: the tile's CSR span exceeds the stage; gather from global memory
};

struct Counters {          // per-thread, reduced once per CTA; rare counters (events, suspects) go straight to the trace row
  u32 packets, edges, changed, pending, kL, kJ, kM, views;
  // single-view kernels (tight register cap) keep six of them in three: a thread visits at most
  // MAX_TILES_PER_CTA = 1024 nodes, each adds at most MAX_FANOUT = 8 to a counter — 16 bits hold that
  u32 pe /* packets | edges << 16 */, cp /* changed | pending << 16 */, kLJ /* kL | kJ << 16 */;
  u64 hash;
};

__device__ __forceinline__ u32 warp_sum(u32 v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ u64 warp_sum64(u64 v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Deliver one entry to `dst` (global id): local → RED.MAX into this shard's inbox plane `plane`
// (= inbox_wr + (kind·R + slot)·n_local) and mark the destination tile hot for the next tick;
// cross-shard → append to the peer's receive window over NVLink.
// Cross-shard staging: every WARP owns one small buffer per destination shard in shared memory; entries are appended
// with a warp-aggregated shared-memory atomic and a buffer that holds at least 32 entries is copied into the peer's
// window by its own warp — 256+ contiguous bytes over NVLink, one global counter atomic per flush, no CTA barrier
// anywhere (a per-tile CTA-wide flush cost four barriers per tile and made every warp wait for the slowest one).
struct XStage { u64 buf[(BLOCK / 32) * XW_TOTAL]; u32 cnt[BLOCK / 32][MAX_WORLD]; };
// (no integer division on the send path: the sharded kernel issues on every cycle it can — 2.4× the instructions of the unsharded one;
// the staging capacity comes with the parameters, and shard_of uses the reciprocal)
__device__ __forceinline__ u32 xseg(const TickParams& p, u32 shard) { return (shard - (shard > p.snd.rank ? 1u : 0u)) * p.xcap; }

// held: what the sender read from the destination word earlier in this launch (0: nothing read).  The words of the plane only
// grow during a launch (RED.MAX is the only write to the planes a launch sends into), so held ≥ val1 means the word already is,
// and will stay, at least val1: the RED would change nothing and is not issued.  The tile is marked all the same.
template <bool SHARDED>
__device__ __forceinline__ void deliver(const TickParams& p, XStage* xs, u32* plane, u32 dst, u32 kind, u32 s, u32 val1, u64 pol_last, bool mark, u32 held = 0) {
  const u32 dl = dst - p.first;
  if (!SHARDED || dl < p.n_local) {
    if (val1 > held) red_max_resident(plane + dl, val1, pol_last);
    else SFS_PROBE(22);
    if (mark) { p.hot_wr[dl >> TILE_SHIFT] = 1; SFS_PROBE(26); }   // sparse ticks only: tell the next tick which tiles received something
  } else {
    const ShardIdx t = shard_of(dst, p.snd.shard_size, p.snd.shard_inv);
    const u32 shard = t.shard;
    const u64 e = win_entry(val1, s + p.sv_wshift, kind, t.local);   // (a single-view launch numbers its view 0: the entry carries the real one)
    // warp-aggregated append: the lanes of this call that target the same shard reserve their slots with ONE
    // shared-memory atomic on the warp's own counter (divergent callers of the same warp may interleave: keep it atomic)
#ifdef SFS_XSTAGE_MATCH                           // A/B: one shared atomic per distinct shard of the call (match_any + leader + shuffle)
    const u32 peers = __match_any_sync(__activemask(), shard);
    const u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5, leader = __ffs(peers) - 1;
    u32 base = 0;
    if (lane == leader) base = atomicAdd(&xs->cnt[wid][shard], (u32)__popc(peers));
    base = __shfl_sync(peers, base, leader);
    const u32 pos = base + (u32)__popc(peers & ((1u << lane) - 1u));
#else                                             // one shared atomic per lane: the hardware serialises the lanes that hit the same counter
    const u32 wid = threadIdx.x >> 5;
    const u32 pos = atomicAdd(&xs->cnt[wid][shard], 1u);
#endif
    if (pos < p.xcap) {
      xs->buf[wid * XW_TOTAL + xseg(p, shard) + pos] = e;
    } else {                                   // buffer full: write this one straight through
      win_append<1>(p.snd, p.overflow, shard, {e});
    }
  }
}

// Unsharded sends of one entry to its first n targets.  With p.dedup (SERFSIM_DEDUP, on by default):  In a saturated tick every sender of a wave
// sends the same value for a (kind, view), and a destination gets about Poisson(fanout) copies: most REDs would write a value the
// word already holds.  The destination words are read first, all together (one round trip per entry, not per target), and only
// the REDs that can raise a word are issued.  Exact whatever the reads return (see deliver).
template <int FMAX>
__device__ __forceinline__ void send_deduped(const TickParams& p, u32* plane, const u32 (&tg)[FMAX], u32 n, u32 val1, u64 pol_last, bool mark) {
  u32 held[FMAX];
#pragma unroll
  for (int k = 0; k < FMAX; ++k) held[k] = ((u32)k < n && p.dedup) ? peek_inbox(plane + (tg[k] - p.first), pol_last) : 0u;
#pragma unroll
  for (int k = 0; k < FMAX; ++k)
    if ((u32)k < n) deliver<false>(p, nullptr, plane, tg[k], 0, 0, val1, pol_last, mark, held[k]);
}

// Copy the warp's staged entries into the peers' windows (whole warp, convergent) in runs of whole 32-entry blocks (256+
// contiguous bytes over NVLink).  Space in a peer's window is reserved with an atomic on this rank's per-peer counter — one
// flush AHEAD: after its blocks have been written, the lane whose index is the peer's rank reserves as many entries as this
// flush used and keeps base and length in its own registers (`resv`, `rlen`); nothing reads them before the next flush, so the
// atomic's round trip on a counter the whole grid hammers is off the critical path (a reservation at flush time, or one issued
// inside the per-peer loop, puts that round trip in front of the next warp shuffle).  In saturated ticks the first reservation is
// made when the kernel starts.  A flush that needs more than it holds takes the rest synchronously.  Reserved entries that stay
// unwritten read as zeros at the receiver: the drain kernel skips zero entries and clears every entry it consumes, so a window
// is all zeros again before it is written next.  force = false: whole blocks only; force = true (end of the kernel): everything.
__device__ __forceinline__ bool flush_xwarp(const TickParams& p, XStage* xs, bool force, u32& resv, u32& rlen) {
  const u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const Sender& x = p.snd;
  __syncwarp();
  bool wrote = false;
  u32 want = 0;                                // this lane's peer: entries to reserve for the next flush
  // peers whose buffer holds a whole block (anything, when forced): lane s looks at peer s, one vote, then only those are visited
  const u32 mine = lane < x.world ? xs->cnt[wid][lane] : 0u;
  u32 ready = __ballot_sync(0xffffffffu, lane != x.rank && (force ? mine != 0 : mine >= XW_FLUSH));
  while (ready) {
    const u32 sh = (u32)__ffs((int)ready) - 1u;
    ready &= ready - 1u;
    const u32 staged = __shfl_sync(0xffffffffu, mine, sh);
    if (staged > p.xcap) wrote = true;        // the excess went straight through
    const u32 n = min(staged, p.xcap);
    const u32 m = force ? n : (n & ~(XW_FLUSH - 1u));          // entries to write now
    u64* src = xs->buf + wid * XW_TOTAL + xseg(p, sh);
    u64* dst = win_segment(x.win_data[sh], x.rank, x.win_cap);
    const u32 base = __shfl_sync(0xffffffffu, resv, sh), avail = __shfl_sync(0xffffffffu, rlen, sh);
    const u32 take = min(m, avail);
    for (u32 i = lane; i < take; i += 32) {
      if (base + i < x.win_cap) dst[base + i] = src[i];
      else *p.overflow = 2;
    }
    if (m > take) {                            // not (enough) reserved ahead: take the rest now
      u32 b2 = 0;
      if (lane == sh) b2 = atomicAdd(x.send_count + sh, m - take);
      b2 = __shfl_sync(0xffffffffu, b2, sh);
      for (u32 i = lane; i < m - take; i += 32) {
        if (b2 + i < x.win_cap) dst[b2 + i] = src[take + i];
        else *p.overflow = 2;
      }
    }
    if (lane == sh) { resv += take; rlen -= take; want = min(m, XW_RESERVE_MAX); }
    wrote = true;
    const u32 rem = n - m;                     // < 32 entries stay staged: move them to the front
    u64 keep = 0;
    if (lane < rem) keep = src[m + lane];
    __syncwarp();
    if (lane < rem) src[lane] = keep;
    if (lane == 0) xs->cnt[wid][sh] = rem;
  }
  // reservations for the next flush: issued last, consumed by the shuffles of the NEXT call
  if (!force && want && rlen == 0) { resv = atomicAdd(x.send_count + lane, want); rlen = want; }
  __syncwarp();
  return wrote;
}

// The gossip peer draw (record.cuh peer_issue) with the neighbour ids requested from the tile's stage or global memory.
template <int FMAX, bool STAGED>
__device__ __forceinline__ void pick_issue(const TickParams& p, const StageView& sv, u32 v, u32 row0, u32 deg, u64 pol_first, u32 (&cand)[FMAX]) {
  peer_issue<FMAX>(p.tick, v, p.fanout, p.seed_lo, p.seed_hi, row0, deg,
                   [&](u32 e) { return (STAGED && sv.col_staged) ? sv.col[e - sv.col_base] : gather_col(p.col + e, pol_first); }, cand);
}

// What decides whether a node has anything to do this tick: its busy byte and the inbox words of the previous tick
// (slot 0 kept; per slot one "has mail" bit), plus — multi-slot runs — one "has queued transmits" bit per slot from the
// queue words.  13 bytes per node instead of 45 (single slot).
// (busy byte: BUSY_*, record.cuh)
// nd: the node's own earliest suspicion deadline (node_due), read only in tiles that have come due
struct Pre { u32 busy, mL, mJ, mM, any, qw, mailmask, qmask, keep, nd; };   // mL, mJ, mM, qw: the words of view `keep` (0 in single-slot runs)
// Carry word of node vl in this tick (CARRY_*), 0 when no earlier pass of the tick visited it.
__device__ __forceinline__ u32 carry_of(const TickParams& p, u32 vl, u64 pol_first) {
  const u32 w = ld_carry(p.carry + vl, pol_first);
  return (w >> 8) == ((p.tick + 1u) & (CARRY_TICKS - 1u)) ? (w & 0xffu) : 0u;
}
template <bool R1, bool PASS = false>
__device__ __forceinline__ Pre prefetch_node(const TickParams& p, u32 vl, bool kL, bool kJ, bool kM, u64 pol_first, bool due, u32 keep = 0) {
  // R1: the kernel visits exactly one view, the one its planes start with (single-slot runs; single-view ticks of multi-slot runs, whose
  // parameter block points at the active view — the distance between the planes of two kinds is p.R views either way)
  const u32 nl = p.stride, R = p.R, s_hi = R1 ? 1u : R;
  Pre x;
  x.busy = ld_busy(p.busy + vl, pol_first);
  x.nd = (!R1 && due) ? ld_node_due(p.node_due + vl, pol_first) : NO_DEADLINE;    // single-view kernels (tight register cap) read it where it is needed instead: one register less across the tile loop
  x.keep = R1 ? 0u : keep;
  x.mL = x.mJ = x.mM = x.qw = 0; x.any = 0; x.mailmask = 0; x.qmask = 0;
  for (u32 s2 = 0; s2 < s_hi; ++s2) {
    const u32 l = kL ? ld_u32_stream(p.inbox_rd + (size_t)(KIND_LEAVE * R + s2) * nl + vl, pol_first) : 0u;
    const u32 j = kJ ? ld_u32_stream(p.inbox_rd + (size_t)(KIND_JOIN * R + s2) * nl + vl, pol_first) : 0u;
    const u32 m = kM ? ld_u32_stream(p.inbox_rd + (size_t)(KIND_ML * R + s2) * nl + vl, pol_first) : 0u;
    const u32 q = ld_qword(p.qword + (size_t)s2 * nl + vl, pol_first);        // queue word (transmit budgets)
    SFS_COUNT(6, 4);
    if (R1 || s2 == x.keep) { x.mL = l; x.mJ = j; x.mM = m; x.qw = q; }
    x.any |= l | j | m;
    x.mailmask |= ((l | j | m) ? 1u : 0u) << s2;
    x.qmask |= (q ? 1u : 0u) << s2;
  }
  // A pass cannot trust busy bits 0 and 3 (an earlier pass of the tick rewrote them): a queued transmit is business of the view itself,
  // and a node whose timers were due when the tick began visits every view (`any` stands for both in the activity test).
  if (PASS) x.any |= x.qw | ((due && (carry_of(p, vl, pol_first) & CARRY_TDUE)) ? 1u : 0u);
  return x;
}
// Has the node anything to do this tick?  (due: its tile's earliest suspicion deadline has been reached — then a node that runs timers
// looks at its OWN earliest deadline: only if that has been reached too does it visit its views; otherwise it hands the deadline back
// to the timer wheel, sleeping_deadline(), without touching a record.)
// A pass does not look at the awake bit (busy bit 0): it says that SOME view of the node keeps a queue or a watcher's probe duty.  The
// pass's own view's queue is in `any` (its queue word), probe duty comes with the static watcher bit 2, and a view with neither, no mail,
// no host operation and no timer due has nothing to do: the view loop leaves it unvisited too.  So a pass skips the nodes that are
// awake only for another view's sake (in a tick in which one view's wave keeps nearly every node awake, nearly all of them).
template <bool PASS = false>
__device__ __forceinline__ u32 busy_business(u32 busy) { return busy & (BUSY_OP | BUSY_WATCH | (PASS ? 0u : BUSY_AWAKE)); }
template <bool PASS = false>
__device__ __forceinline__ bool node_active(const TickParams& p, const Pre& x, bool due) {
  return busy_business<PASS>(x.busy) != 0 || x.any != 0 || p.reap_now != 0 || (due && (x.busy & BUSY_TIMER) && x.nd <= p.tick);
}

// Multi-slot runs, saturated ticks: what a node needs beyond its `Pre` words, requested ONE TILE AHEAD together with them — the node
// word, the neighbour ids of its gossip peers (uniform out-degree: the row offset is arithmetic, the draw needs only tick and id) and the
// record of the view it will most probably visit first (`keep`: the first view this thread visited in its previous tile; in a
// dissemination wave nearly every node has the same views active).  The multi-slot kernel holds 8 warps per SM (one CTA of 256 threads,
// ≈ 200 registers per thread): without this every tile pays three dependent round trips (Pre → node word + record → neighbour ids) with too few warps to
// hide them.  A guess that turns out wrong costs one unused 32-byte load; results never depend on it.
template <int FMAX>
struct Ahead { u64 ns; Words rec; u32 cand[FMAX]; u32 valid; };

__device__ __forceinline__ u32 sleeping_deadline(const Pre& x, bool due) { return (due && (x.busy & BUSY_TIMER)) ? x.nd : NO_DEADLINE; }

// ---- cold paths of a node's tick, kept out of line: host operations, the reaper round and the SWIM probe run for a handful of
// nodes per tick (or for all of them once in a long while); inlined, their temporaries (a second Philox block, the operation
// scan) raise the register demand of the path every node takes and make it spill.  They are called on COPIES of the view and
// the node's scalars: a variable whose address is passed to a call lives in local memory for its whole lifetime, and the
// hot path's record must stay in registers (measured: 4.6 extra L2 sectors per node and +25 % per plateau tick otherwise).
#if defined(SFS_COLD_INLINE)
#define SFS_COLD __forceinline__               // A/B: everything inline again
#elif defined(SERFSIM_EMU)
#define SFS_COLD __attribute__((noinline))
#else
#define SFS_COLD __noinline__
#endif
// Phase E — what the API call does at its origin (SURVEY Appendix A.8): Serf::join / leave / remove_failed_node[_prune], crash, restart.
__device__ SFS_COLD void cold_host_op(Rec& r, u32& clock, u32& sstate, u32 op, bool op_here, bool self, bool up_r, u32 limit) {
  if (op == OP_REJOIN && self && !up_r) {
    r.inc += 1; r.mlstate = ML_ALIVE; r.qfrom = 0; r.txm = limit; r.deadline = 0; r.mask = 0;
    sstate = SS_ALIVE;
    node_join(r);
  }
  if (((op == OP_JOIN && up_r) || (op == OP_REJOIN && !up_r)) && self) {     // serf/api.rs:339-342 → serf/base.rs:381-397
    const u32 T = clock; witness(clock, T);
    join_intent(r, T, limit);
    r.qjoin = T; r.txj = limit;
  }
  if (op == OP_LEAVE && up_r && self && sstate == SS_ALIVE) {                // serf/api.rs:422-449
    sstate = SS_LEAVING;
    const u32 T = clock; clock += 1;
    bool rf = false;
    leave_intent(r, T, false, true, sstate, rf, limit);
    r.qleave = T; r.txl = limit; r.flags &= ~FLAG_QPRUNE;
  }
  if ((op == OP_FORCE_LEAVE || op == OP_FORCE_LEAVE_PRUNE) && up_r && op_here) {   // serf/base.rs:454-480 (remove_failed_node[_prune], serf/api.rs:500-515)
    const u32 T = clock; witness(clock, T);
    const bool prune = op == OP_FORCE_LEAVE_PRUNE;
    bool rf = false;
    leave_intent(r, T, prune, self, sstate, rf, limit);
    r.qleave = T; r.txl = limit; r.flags = (r.flags & ~FLAG_QPRUNE) | (prune ? FLAG_QPRUNE : 0u);   // queued whatever the handler said
    if (rf) { const u32 T2 = clock; witness(clock, T2); join_intent(r, T2, limit); r.qjoin = T2; r.txj = limit; }
  }
}
// Which host operation targets node v this tick?
__device__ SFS_COLD u32 cold_find_op(const TickParams& p, u32 v, u32& op_slot) {
  atomicAdd((unsigned long long*)(p.row + ROW_EVENTS), 1ull);
  return host_op_of(p, v, op_slot);
}
// Reaper round (serf/base.rs:483-610): Left / Failed members past their timeouts are erased, stale buffered intents dropped.
__device__ SFS_COLD void cold_reap(Rec& r, u32 t, u32 tombstone, u32 reconnect, u32 intent) {
  const u32 age = r.leave_tick ? (t + 1 - r.leave_tick) : 0;
  if ((r.flags & 1) && r.leave_tick && ((r.status == ST_LEFT && age > tombstone) || (r.status == ST_FAILED && age > reconnect))) {
    r.flags &= ~1u; r.status = TY_NONE; r.st = 0; r.leave_tick = 0;           // erase_node! :499-519
    SFS_PROBE(27);
  } else if (!(r.flags & 1) && r.status != TY_NONE && r.leave_tick && age > intent) {
    r.status = TY_NONE; r.st = 0; r.leave_tick = 0;                           // reap_intents :1817-1822
  }
}
// SWIM probe target of a watcher's round: a uniformly random neighbour (memberlist walks a shuffled list).
__device__ SFS_COLD u32 cold_probe_target(const TickParams& p, u32 v, u32 row0, u32 deg) {
  return __ldg(p.col + row0 + neighbour_slot(p.tick, v, DOMAIN_PROBE, p.seed_lo, p.seed_hi, deg));
}
// The probe found the subject down: suspect it (or confirm with this node's bucket).
__device__ SFS_COLD void cold_probe_hit(const TickParams& p, Rec& r, u32 v) {
  if (r.mlstate == ML_ALIVE || r.mlstate == ML_SUSPECT) {
    if (r.mlstate == ML_ALIVE) atomicAdd((unsigned long long*)(p.row + ROW_SUSPECTS), 1ull);
    ml_suspect(r, r.inc, from_bucket(v), p.tick, false, p.rules);
  }
}
// The view rules of record.cuh that only a few views need in a tick
__device__ SFS_COLD void cold_refute(Rec& r, u32& clock, u32 limit) { refute_leave(r, clock, limit); }
__device__ SFS_COLD bool cold_can_confirm(u32 k, u32 mask, u32 v) { return can_confirm(k, mask, v); }

// Returns true when the node stays awake (queued transmits, probe duty): that keeps its tile hot for the next tick.
// A view whose only business is a running suspicion timer does not: its deadline goes to `mind` (the caller registers the
// minimum in tile_due) and the view sleeps until its tile comes due.  `due`: this tile's earliest deadline has been reached —
// every node of it that carries a timer (busy bit 3) visits all its views.
template <bool TRACE, int FMAX, bool SHARDED, bool R1, bool STAGED, bool PASS = false>
__device__ __forceinline__ bool process_node(const TickParams& p, const StageView& sv, XStage* xs, const u32 vl, const Pre& pre, const bool kL, const bool kJ, const bool kM, const bool mark, const bool saturated,
                                             const bool due, const u64 pol_first, const u64 pol_last, Counters& c, u32& mind, int& dsusp, const Ahead<FMAX>& ah, u32& first_view, const u32 sv_views = 0xffffffffu,
                                             const bool carry_out = false) {
  static_assert(!STAGED || R1, "the staged path is the single-slot path");
  static_assert(!PASS || (R1 && !STAGED && !SHARDED && !TRACE), "passes are single-slot kernels of unsharded production runs");
  const u32 lt = threadIdx.x;              // index inside the staged tile
  const u32 v = p.first + vl;
  const u32 t = p.tick;
  const u32 limit = p.rules.limit;
  const u32 nl = p.stride;               // plane stride (n_local rounded up to a whole tile)
  const u32 R = p.R;                     // R1: one view is visited, the first of the planes as this launch sees them (they keep the distance of p.R views between kinds)

  // ---- loads.  Saturated ticks (the previous tick delivered to at least half of the nodes): everything a node
  // needs is requested up front, independent loads in flight together.  Otherwise most nodes are idle: read only
  // the busy byte and the inbox words, and fetch the 8-byte node word and the 32-byte record just for the nodes
  // that have something to do.  Multi-slot runs fetch the records of the views that have something to do. ----
  const bool upfront = R1 && (saturated || TRACE || STAGED);
  u64 ns = 0;
  u32 row0 = 0, row1 = 0;
  Words cur;
  auto load_node = [&]() {
    ns = STAGED ? sv.node[lt] : ld_u64_stream(p.node_state + vl, pol_first);
    if (STAGED) { row0 = sv.rowptr[lt]; row1 = sv.rowptr[lt + 1]; }
    else if (p.udeg) { row0 = vl * p.udeg; row1 = row0 + p.udeg; }     // uniform out-degree: the row offsets are arithmetic
    else { row0 = ld_row_ptr(p.row_ptr + vl, pol_first); row1 = ld_row_ptr(p.row_ptr + vl + 1, pol_first); }
  };
  auto load_rec0 = [&]() {
    if (STAGED) {
      const uint4 a = reinterpret_cast<const uint4*>(sv.rec + lt)[0], b = reinterpret_cast<const uint4*>(sv.rec + lt)[1];
      cur.w[0] = a.x; cur.w[1] = a.y; cur.w[2] = a.z; cur.w[3] = a.w; cur.w[4] = b.x; cur.w[5] = b.y; cur.w[6] = b.z; cur.w[7] = b.w;
    } else {
      cur = ld_rec256(p.rec + 2 * (size_t)vl, pol_first);
    }
    merge_queue_word(cur, pre.qw);                         // the record image everything below works on is record | budgets
  };
  if (upfront) { load_node(); load_rec0(); }
  const u32 busy = pre.busy;
  u32 mL = pre.mL, mJ = pre.mJ, mM = pre.mM;
  if (STAGED) { mL = kL ? sv.inL[lt] : 0u; mJ = kJ ? sv.inJ[lt] : 0u; mM = kM ? sv.inM[lt] : 0u; }

  // ---- idle exit: nothing received (any slot), nothing queued, no host operation, no probe duty, no timer due ----
  u32 nd = pre.nd;                                       // the node's own earliest deadline: matters in due tiles, for nodes that run timers
  if (R1 && due && (busy & BUSY_TIMER)) nd = ld_node_due(p.node_due + vl, pol_first);
  const u32 sleeping = (due && (busy & BUSY_TIMER)) ? nd : NO_DEADLINE;
  bool timers_due = sleeping <= p.tick;
  u32 cr = 0;                                            // PASS: what the earlier passes of this tick did at this node
  if (PASS && due) { cr = carry_of(p, vl, pol_first); if (cr & CARRY_SEEN) timers_due = (cr & CARRY_TDUE) != 0; }   // as it was when the tick began
  if (!TRACE && !STAGED && !(busy_business<PASS>(busy) != 0 || pre.any != 0 || p.reap_now != 0 || timers_due)) { mind = min(mind, sleeping); if (due && (busy & BUSY_TIMER)) SFS_PROBE(20); return false; }
  if (PASS && !due) cr = carry_of(p, vl, pol_first);
  if (STAGED && !TRACE && !(busy_business(busy) || (mL | mJ | mM) || p.reap_now || timers_due)) { mind = min(mind, sleeping); return false; }
  // (the watcher mask — subjects this node can probe, it has them as neighbours — is re-read where a watcher needs it: a handful of nodes)
#define SFS_WMASK() ((busy & BUSY_WATCH) ? (ld_watch(p.watch + vl, pol_first) >> p.sv_wshift) : 0u)   /* sv_wshift: the view a single-view launch works on (0 in every other launch) */
  const bool ahead = !R1 && !STAGED && ah.valid;       // node word, peers' ids and the record of view pre.keep were requested a tile ago
  if (ahead) { ns = ah.ns; row0 = vl * p.udeg; row1 = row0 + p.udeg; }
  else if (!upfront) { load_node(); if (R1) load_rec0(); }

  u32 clock = nw_clock(ns);
  const bool up_r = nw_up(ns);
  u32 sstate = nw_sstate(ns);
  const u32 deg = row1 - row0;

  // host operation for this node (at most one per tick)
  u32 op = 0, op_slot = 0;
  if (busy & BUSY_OP) { u32 slot_tmp = 0; op = cold_find_op(p, v, slot_tmp); op_slot = slot_tmp; }
  bool up_s = up_r;
  if (op == OP_FAIL) up_s = false;
  if (op == OP_REJOIN) up_s = true;

  // SWIM probe target of this round (only matters while some tracked subject is down)
  bool have_probe = false;
  u32 ptarget = 0;
  if (up_s && (busy & BUSY_WATCH) && p.probe_every && p.down_mask && ((t + v) % p.probe_every) == 0 && deg) {
    ptarget = (STAGED && sv.col_staged) ? 0u : cold_probe_target(p, v, row0, deg);
    if (STAGED && sv.col_staged) ptarget = sv.col[row0 + neighbour_slot(t, v, DOMAIN_PROBE, p.seed_lo, p.seed_hi, deg) - sv.col_base];
    have_probe = true;
  }

  u32 tg[FMAX];
  u32 nt = 0;
  bool have_targets = false;
  u32 max_tx = 0;
  bool awake = false, has_timer = false, dl_moved = false;
  // (`mind`, NO_DEADLINE on entry: the earliest running suspicion deadline among the views visited)

  // Views to visit: all of them when the node as a whole has business (trace, reaper round, host operation, timers due);
  // otherwise those with mail, queued transmits or probe duty (a watcher's view of a subject that is down).
  const u32 all_views = (R >= 32u) ? 0xffffffffu : ((1u << R) - 1u);
  const bool visit_all = R1 || TRACE || p.reap_now || (busy & BUSY_OP) || timers_due || !p.sleep_on;
  u32 todo = visit_all ? all_views : ((pre.mailmask | pre.qmask | (p.probe_every ? (SFS_WMASK() & p.down_mask) : 0u)) & all_views);
  if (!R1) SFS_COUNT(5, R - (u32)__popc(todo));             // views left asleep by a visited node

  // multi-slot runs: the record and inbox words of the next view to visit are requested while the current one is processed
  Words nxt = {};
  u32 nL = 0, nJ = 0, nM = 0, nq = 0;
  auto load_view = [&](u32 s2, Words& w, u32& q, u32& iL, u32& iJ, u32& iM) {
    const size_t idn = (size_t)s2 * nl + vl;
    w = ld_rec256(p.rec + 2 * idn, pol_first);
    if (s2 == pre.keep) { q = pre.qw; iL = pre.mL; iJ = pre.mJ; iM = pre.mM; return; }
    q = ld_qword(p.qword + idn, pol_first);
    SFS_COUNT(6, 4);
    iL = kL ? ld_u32_stream(p.inbox_rd + (size_t)(KIND_LEAVE * R + s2) * nl + vl, pol_first) : 0;
    iJ = kJ ? ld_u32_stream(p.inbox_rd + (size_t)(KIND_JOIN * R + s2) * nl + vl, pol_first) : 0;
    iM = kM ? ld_u32_stream(p.inbox_rd + (size_t)(KIND_ML * R + s2) * nl + vl, pol_first) : 0;
  };
#ifndef SFS_VIEW_PREFETCH
#define SFS_VIEW_PREFETCH 0                  // 1: the next view's record is requested while the current one is processed (12 more live registers; measured slower)
#endif
  u32 s = R;
  if (R1) { s = 0; todo = 0; }
  else if (todo) {
    s = (u32)__ffs((int)todo) - 1u; todo &= todo - 1u;
    u32 q0;
    if (ahead && s == pre.keep) { cur = ah.rec; q0 = pre.qw; mL = pre.mL; mJ = pre.mJ; mM = pre.mM; SFS_PROBE(18); }
    else load_view(s, cur, q0, mL, mJ, mM);
    merge_queue_word(cur, q0);
    first_view = s;
  }
#pragma unroll 1
  while (s < R) {
    const size_t idx = (size_t)s * nl + vl;
    u32 s_next = R;
    if (!R1 && todo) { s_next = (u32)__ffs((int)todo) - 1u; todo &= todo - 1u; if (SFS_VIEW_PREFETCH) load_view(s_next, nxt, nq, nL, nJ, nM); }
    if (mL) st_u32_stream(p.inbox_rd + (size_t)(KIND_LEAVE * R + s) * nl + vl, 0u, pol_first);   // consume: clear for reuse in two ticks
    if (mJ) st_u32_stream(p.inbox_rd + (size_t)(KIND_JOIN * R + s) * nl + vl, 0u, pol_first);
    if (mM) st_u32_stream(p.inbox_rd + (size_t)(KIND_ML * R + s) * nl + vl, 0u, pol_first);
    const Words orig = cur;
    Rec r;
    unpack(cur, r);
    const bool self = (p.subj[s] == v);
    const bool susp_before = up_r && r.mlstate == ML_SUSPECT;
    if (!R1 && p.sv_mode == SV_CHECK && !((sv_views >> s) & 1u) && up_r &&
        ((mL | mJ | mM) || (r.txl | r.txj | r.txm) || r.mlstate == ML_SUSPECT)) *p.overflow = 4;     // SERFSIM_SV=2: the set of views with business was not a superset

    // ---------------- Phase R ----------------
    if (up_r && (mL | mJ | mM)) {
      if (mM) {
        const u32 key = mM - 1, inc = ml_key_inc(key), kind = ml_key_state(key), fromb = ml_key_from(key);
        if (kind == ML_ALIVE) ml_alive(r, inc, self, limit);
        else if (kind == ML_SUSPECT) ml_suspect(r, inc, fromb, t, self, p.rules);
        else ml_dead(r, inc, kind == ML_LEFT, t, self, limit);
      }
      bool refute = false;
      if (mL) { const u32 key = mL - 1, lt = leave_key_lt(key); witness(clock, lt); leave_intent(r, lt, leave_key_prune(key), self, sstate, refute, limit); }
      if (mJ) { const u32 lt = mJ - 1; witness(clock, lt); join_intent(r, lt, limit); }
      if (refute) { Rec tr = r; u32 ck = clock; cold_refute(tr, ck, limit); r = tr; clock = ck; }
      stamp_intent(r, orig, t);
      Words mid;
      pack(r, mid);
      if (R1) c.cp += differs(mid, orig) ? 1u : 0u; else c.changed += differs(mid, orig) ? 1 : 0;
    }
    // ---------------- Phase E ----------------
    if (op) { Rec tr = r; u32 ck = clock, ss = sstate; cold_host_op(tr, ck, ss, op, op_slot == s, self, up_r, limit); r = tr; clock = ck; sstate = ss; }
    if (op && !(r.flags & 1) && r.status != TY_NONE && r.leave_tick == 0) r.leave_tick = t + 1;
    if (up_s) {
      // ---------------- Phase T: reaper (serf/base.rs:483-610), suspicion timer, probe ----------------
      if (p.reap_now) { Rec tr = r; cold_reap(tr, t, p.tombstone_ticks, p.reconnect_ticks, p.intent_ticks); r = tr; }
      if (r.mlstate == ML_SUSPECT && r.deadline != 0 && t >= r.deadline) ml_dead(r, r.inc, false, t, false, limit);
      if (have_probe && !self && ptarget == p.subj[s] && ((p.down_mask >> s) & 1)) { Rec tr = r; cold_probe_hit(p, tr, v); r = tr; }
      // ---------------- Phase S ----------------
      const u32 mx = max(r.txl, max(r.txj, r.txm));
      if (mx) {
        if (!have_targets) {
          if (ahead) nt = peer_finish<FMAX>(v, ah.cand, tg);
          else {
            u32 cand[FMAX];
            pick_issue<FMAX, STAGED>(p, sv, v, row0, deg, pol_first, cand);
            nt = peer_finish<FMAX>(v, cand, tg);
          }
          have_targets = true;
        }
        u32* const planeL = p.inbox_wr + (size_t)(KIND_LEAVE * R + s) * nl;
        u32* const planeJ = p.inbox_wr + (size_t)(KIND_JOIN * R + s) * nl;
        u32* const planeM = p.inbox_wr + (size_t)(KIND_ML * R + s) * nl;
        const u32 vL = leave_key(r.qleave, (r.flags & FLAG_QPRUNE) != 0) + 1, vJ = r.qjoin + 1, vM = ml_key(r) + 1;
        const u32 sL = min(r.txl, nt), sJ = min(r.txj, nt), sM = min(r.txm, nt);     // entry e goes to targets 0 .. min(tx_e, nt)-1
        if (!SHARDED) {
          send_deduped<FMAX>(p, planeL, tg, sL, vL, pol_last, mark);
          send_deduped<FMAX>(p, planeJ, tg, sJ, vJ, pol_last, mark);
          send_deduped<FMAX>(p, planeM, tg, sM, vM, pol_last, mark);
        } else {
#pragma unroll
          for (int k = 0; k < FMAX; ++k) {
            if ((u32)k < sL) deliver<SHARDED>(p, xs, planeL, tg[k], KIND_LEAVE, s, vL, pol_last, mark);
            if ((u32)k < sJ) deliver<SHARDED>(p, xs, planeJ, tg[k], KIND_JOIN, s, vJ, pol_last, mark);
            if ((u32)k < sM) deliver<SHARDED>(p, xs, planeM, tg[k], KIND_ML, s, vM, pol_last, mark);
          }
        }
        if (R1) { c.kLJ += sL | (sJ << 16); c.kM += sM; c.pe += min(mx, nt) << 16; }
        else { c.kL += sL; c.kJ += sJ; c.kM += sM; c.edges += min(mx, nt); }
        max_tx = max(max_tx, mx);
        r.txl -= sL; r.txj -= sJ; r.txm -= sM;
      }
      // Serf::leave: our own leave intent is out → memberlist.leave() → dead{node == from}  (serf/api.rs:451-476)
      if (self && sstate == SS_LEAVING && r.txl == 0 && r.mlstate == ML_ALIVE) {
        r.mlstate = ML_LEFT; r.qfrom = 0; r.txm = limit; sstate = SS_LEFT;
      }
      // Suspect views are counted in `pending` by the persistent counter (they sleep), the others here.
      if ((!R1 || PASS) && (rec_queued(r) || mx)) c.views |= 1u << (s + p.sv_slot * PASS);   // the view sent mail or keeps a queue: it has business in the next tick (passes, single-view ticks)
      // (view_watching / view_pending / view_awake of record.cuh, written out: through the helpers this kernel takes 32 more instructions)
      const bool queued = rec_queued(r);
      const bool watching = (busy & BUSY_WATCH) && p.probe_every && ((p.down_mask >> s) & 1) && !self && ((SFS_WMASK() >> s) & 1);
      const bool suspect = r.mlstate == ML_SUSPECT;
      { const u32 pnd = (!suspect && (queued || (watching && r.mlstate == ML_ALIVE))) ? 1u : 0u; if (R1) c.cp += pnd << 16; else c.pending += pnd; }
      awake |= queued || (watching && (r.mlstate == ML_ALIVE || (suspect && cold_can_confirm(p.rules.k, r.mask, v))));
      if (suspect && r.deadline != 0) { has_timer = true; mind = min(mind, r.deadline); dl_moved |= r.deadline != orig.w[4]; }
    }
    dsusp += ((up_s && r.mlstate == ML_SUSPECT) ? 1 : 0) - (susp_before ? 1 : 0);
    pack(r, cur);
    {
      Words o2 = orig, c2 = cur;                           // storage image: record without budgets, budgets in the queue word
      const u32 q_old = split_queue_word(o2), q_new = split_queue_word(c2);
      if (differs(c2, o2)) st_rec256(p.rec + 2 * idx, c2, pol_first);
      if (q_new != q_old) { st_qword(p.qword + idx, q_new, pol_first); SFS_COUNT(7, 4); }
    }
    if (TRACE) c.hash += rec_hash((u64)s * p.n_global + v, cur);
    if (r.inc >= INC_LIMIT) *p.overflow = 1;
    if (!R1) {
      if (!SFS_VIEW_PREFETCH && s_next < R) load_view(s_next, nxt, nq, nL, nJ, nM);
      cur = nxt; merge_queue_word(cur, nq); mL = nL; mJ = nJ; mM = nM;
    }
    s = s_next;
  }
  const u64 ns2 = node_word(clock, up_s, sstate);
  if (ns2 != ns) st_u64_stream(p.node_state + vl, ns2, pol_first);
  if (TRACE) c.hash += node_hash((u64)R * p.n_global + v, ns2);
  if (clock >= LTIME_LIMIT) *p.overflow = 1;
  // packets: min(#peers, the largest budget of any view) — a pass counts what the earlier passes of the tick have not
  const u32 pk = min(nt, max_tx), pk_before = PASS ? (cr & CARRY_PK) : 0u;
  if (R1) c.pe += pk > pk_before ? pk - pk_before : 0u; else c.packets += pk;
  const bool awake_node = awake || (PASS && (cr & CARRY_AWAKE));
  // What a visit of every view makes exact.  A pass sees every view of a node whose timers were due only together with the other passes
  // of the tick: the first pass that visits it writes exactly, the later ones add to what it wrote.
  const bool exact = PASS ? (timers_due && !(cr & CARRY_SEEN)) : visit_all;
  // busy byte: the op bit is consumed, the watcher bit is static; the timer bit is exact after a visit of every view and
  // sticky otherwise (a view that was not visited may run a timer: it is found when its tile comes due)
  const u32 busy2 = (awake_node ? BUSY_AWAKE : 0u) | (busy & BUSY_WATCH) | ((has_timer || (!exact && (busy & BUSY_TIMER))) ? BUSY_TIMER : 0u);
  if (busy2 != busy) st_busy(p.busy + vl, busy2, pol_first);
  // node_due: a lower bound of the node's earliest running deadline, exact after a visit of every view.  A view's deadline only moves
  // while the view is visited, so views that were not visited are still covered by the word as it stands (in a pass: unless an earlier
  // pass rewrote the word exactly).
  if (has_timer) {
    if (exact || !(busy & BUSY_TIMER)) st_node_due(p.node_due + vl, mind, pol_first);
    else if (dl_moved || (PASS && (cr & CARRY_TDUE))) atomicMin(p.node_due + vl, mind);
  }
  if (PASS ? !timers_due : !visit_all) mind = min(mind, sleeping);   // its tile's entry was reset: timers of the views not visited go back with the node's word
  if (PASS && carry_out)                                 // a later pass of this tick has business
    st_carry(p.carry + vl, (((p.tick + 1u) & (CARRY_TICKS - 1u)) << 8) | CARRY_SEEN | (timers_due ? CARRY_TDUE : 0u) | (awake_node ? CARRY_AWAKE : 0u) | max(pk, pk_before), pol_first);
  // The scheduler must know whether anybody stays awake.  A node that sent a packet this tick shows in the row's message count;
  // the others (a watcher on probe duty, a queue that has no peer to go to, a transmit queued after the send phase) are rare.
  // (a pass counts the node when its own view leaves it awake without a packet: more often than the view loop would only if a packet was
  // sent in the tick, and then the row's message count keeps the cluster awake anyway)
  if (awake && pk == 0) atomicAdd(p.sched + SCHED_AWAKE, 1u);
  return awake;
}

__device__ __forceinline__ u32 warp_min(u32 v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// After a warp has processed its nodes of one tile: register the earliest running suspicion deadline in the timer wheel and add
// the warp's net change of Suspect views to the CTA's shared counter (both rare outside suspicion waves: one vote each).
__device__ __forceinline__ void note_timers(const TickParams& p, u32 tile, u32 mind, int dsusp, int* dsusp_s) {
  if (!__any_sync(0xffffffffu, (mind != NO_DEADLINE) | (dsusp != 0))) return;      // one vote on the common path
  const u32 wm = warp_min(mind);
  const u32 ws = warp_sum((u32)dsusp);                     // two's complement: the sum of the lanes' signed changes
  if ((threadIdx.x & 31) == 0) {
    if (wm != NO_DEADLINE) atomicMin(p.tile_due + tile, wm);
    if (ws) atomicAdd(dsusp_s, (int)ws);
  }
}

// A skipped tick (tick_is_idle): nothing can happen, so the only trace it leaves is its row — nothing delivered, nothing
// changed, `pending` = the sleeping Suspect views, and (trace runs) the state hash of the previous tick.
template <bool TRACE>
__device__ __forceinline__ void write_idle_row(const TickParams& p) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    SFS_PROBE(3);                                          // skipped ticks
    p.row[ROW_PENDING] += *reinterpret_cast<const u64*>(p.sched + SCHED_SUSPECTS);
    if (TRACE && p.tick > 0) p.row[ROW_HASH] = *(p.row - ROW_FIELDS + ROW_HASH);
  }
}

// Scan of the CTA's tile flags.  hot_s[i]: bit 0 = process the tile, bit 1 = its earliest suspicion deadline has been reached
// (the entry is reset here, by the tile's owner, before any of its nodes runs: the timers that are still running re-register).
// keep (first of several passes): the flags are replaced by the decision instead of being consumed; the later passes read it (tile_decisions).
__device__ __forceinline__ void scan_tiles(const TickParams& p, u8* hot_s, u32 tile0, u32 ntile, bool all_hot, bool keep = false) {
  for (u32 i = threadIdx.x; i < ntile; i += BLOCK) {
    const u8 f = p.hot_rd[tile0 + i];
    const bool due = p.tile_due[tile0 + i] <= p.tick;
    if (due) { p.tile_due[tile0 + i] = NO_DEADLINE; SFS_PROBE(4); }     // tiles woken by the timer wheel
    const u8 d = (u8)(((f || all_hot || due || p.hot_static[tile0 + i]) ? 1u : 0u) | (due ? 2u : 0u));
    hot_s[i] = d;
    if (keep ? d != f : f != 0) p.hot_rd[tile0 + i] = keep ? d : 0;   // consumed; this parity is written again two ticks from now
  }
}
// Later passes of a tick: the first pass's decision (nothing to process for a pass without business); the last pass consumes it.
__device__ __forceinline__ void tile_decisions(const TickParams& p, u8* hot_s, u32 tile0, u32 ntile, bool last, bool work) {
  for (u32 i = threadIdx.x; i < ntile; i += BLOCK) {
    const u8 d = p.hot_rd[tile0 + i];
    hot_s[i] = work ? d : (u8)0;
    if (last && d) p.hot_rd[tile0 + i] = 0;
  }
}

// What publish_kernel does, for one peer per calling thread (threads 0 .. world-1 of one CTA): entry count, this rank's trace row and
// scheduler verdict into the peer's control block, then the release flag of this exchange.
__device__ __forceinline__ void publish_to_peer(u32 r, u32 world, u32 rank, u32 xpar, u32 stamp, u32 loopback, u32* const* peer_ctrl, u32* send_count,
                                                const volatile u64* row, const volatile u32* sched) {
  if (r >= world || r == rank) return;
  const u32 me = loopback ? r : rank;                       // the slot this rank owns in the peer's control block
  u32* const ctrl = peer_ctrl[r];
  ctrl_counts(ctrl, xpar)[me] = send_count[r];
  u64* sums = ctrl_sums(ctrl, xpar)[me];
#pragma unroll
  for (int i = 0; i < ROW_FIELDS; ++i) sums[i] = row[i];              // this rank's counters of the tick: every rank sums them on the device
  sums[CTRL_QUIET] = sched[SCHED_LOCAL_QUIET]; sums[CTRL_UNTIL] = sched[SCHED_LOCAL_UNTIL]; sums[CTRL_VIEWS] = sched[SCHED_VIEWS_NEW];
  __threadfence_system();
  st_release_sys(ctrl_flags(ctrl, xpar) + me, stamp);
  send_count[r] = 0;
}

// End of a tick: block reduction of the counters (warp shuffles, then shared memory) → one atomic per counter per CTA; the
// LAST CTA to finish (ticket) completes the row and decides how long the cluster can sleep.
// trace row: the first five fields (ROW_PACKETS .. ROW_PENDING) from the counters, (events, suspects: direct), hash
template <bool TRACE, bool PACKED, bool PASS = false>
__device__ __forceinline__ void finish_tick(const TickParams& p, const Counters& c, u64 (*red)[BLOCK / 32], int dsusp_cta) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __shared__ u32 last_s, due_min_s[BLOCK / 32];
  const u32 kL = PACKED ? (c.kLJ & 0xffffu) : c.kL, kJ = PACKED ? (c.kLJ >> 16) : c.kJ;
  const u64 vals[8] = {PACKED ? (c.pe & 0xffffu) : c.packets, PACKED ? (c.pe >> 16) : c.edges, (u64)kL + kJ + c.kM, PACKED ? (c.cp & 0xffffu) : c.changed,
                       PACKED ? (c.cp >> 16) : c.pending, kL, kJ, c.kM};
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const u32 s = warp_sum((u32)vals[i]);
    if (lane == 0) red[i][wid] = s;
  }
  u64 hs = 0;
  if (TRACE) hs = warp_sum64(c.hash);
  __syncthreads();                                         // dsusp_cta is complete
  if (threadIdx.x == 0 && dsusp_cta) atomicAdd(reinterpret_cast<unsigned long long*>(p.sched + SCHED_SUSPECTS), (unsigned long long)(long long)dsusp_cta);
  if (threadIdx.x < 8) {
    u64 s = 0;
#pragma unroll
    for (int w = 0; w < BLOCK / 32; ++w) s += red[threadIdx.x][w];
    if (s) {
      if (threadIdx.x < ROW_EVENTS) atomicAdd((unsigned long long*)(p.row + threadIdx.x), (unsigned long long)s);
      else {
        atomicAdd(p.kinds_cur + (threadIdx.x - 5), (u32)min(s, (u64)0xffffffffu));
        if (PASS) atomicAdd(p.view_kinds_cur + (threadIdx.x - 5), (u32)min(s, (u64)0xffffffffu));   // a pass counts its own view only
      }
    }
  }
  if (TRACE && lane == 0 && hs) atomicAdd((unsigned long long*)(p.row + ROW_HASH), (unsigned long long)hs);
  { const u32 vw = __reduce_or_sync(0xffffffffu, c.views); if (lane == 0 && vw) atomicOr(p.sched + SCHED_VIEWS_NEXT, vw); }
  if (PASS && p.sv_slot + 1u < p.sv_R) return;             // the last pass of the tick completes it
  // ---- ticket: every CTA's counters are in the row before the last one reads it ----
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last_s = (atomicAdd(p.sched + SCHED_TICKET, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (!last_s) return;
  __threadfence();
  volatile u32* sched = p.sched;
  volatile u64* row = p.row;
  const u64 suspects = *reinterpret_cast<volatile u64*>(p.sched + SCHED_SUSPECTS);
  // Can the next ticks do anything?  Not if nothing was sent (no mail), nobody stays awake (no queued transmit, no probe duty),
  // the user-event kernel reported nothing queued or sent (with injectors sleep_on is off): then the cluster sleeps until the earliest
  // suspicion deadline or the next anti-entropy / reaper round (host operations are checked at launch).  Sharded runs: this is
  // the rank's verdict; it travels with the row and the drain kernel combines the ranks' (all quiet, earliest deadline).
  // (decided by ONE thread and broadcast: the words it reads are cleared below by thread 0, and a warp that evaluated them later than
  // thread 0 cleared them would take the other side of a branch that contains a barrier)
  __shared__ u32 quiet_s;
  if (threadIdx.x == 0) quiet_s = (p.sleep_on && row[ROW_EDGES] == 0 && row[ROW_MESSAGES] == 0 && sched[SCHED_AWAKE] == 0 && sched[SCHED_UE_ACTIVITY] == 0) ? 1u : 0u;
  __syncthreads();
  const bool quiet = quiet_s != 0;
  u32 until = p.tick + 1;
  if (quiet) {                                             // uniform over the CTA
    u32 m = NO_DEADLINE;
    for (u32 i = threadIdx.x; i < p.n_tiles; i += BLOCK) m = min(m, __ldcg(p.tile_due + i));
    m = warp_min(m);
    if (lane == 0) due_min_s[wid] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 0; w < BLOCK / 32; ++w) m = min(m, due_min_s[w]);
      // a round runs in tick u when (u + 1) % period == 0; the first such u > tick:
      if (p.pp_every) m = min(m, ((p.tick + 1) / p.pp_every + 1) * p.pp_every - 1);
      if (p.reap_every) m = min(m, ((p.tick + 1) / p.reap_every + 1) * p.reap_every - 1);
      until = max(m, p.tick + 1);
    }
  }
  if (threadIdx.x == 0) {
    row[ROW_PENDING] = row[ROW_PENDING] + suspects;                            // pending = awake views counted above + sleeping Suspect views
    if (p.snd.world == 1) {
      sched[SCHED_IDLE_UNTIL] = until;
      if (p.host_idle_until) *p.host_idle_until = until;
    } else {
      sched[SCHED_LOCAL_QUIET] = quiet ? 1u : 0u; sched[SCHED_LOCAL_UNTIL] = until;
    }
    const u32 awake_n = sched[SCHED_AWAKE];
    sched[SCHED_AWAKE] = 0; sched[SCHED_UE_ACTIVITY] = 0; sched[SCHED_TICKET] = 0;
    // (the single-view kernel keeps no per-thread set: its view has business again iff anything was sent or anybody stays awake)
    const u32 sv_next = (p.sv_mode == SV_SINGLE && (row[ROW_MESSAGES] != 0 || awake_n != 0)) ? (1u << p.sv_slot) : 0u;
    // this tick's set stays readable (OLD) for the kernel of this tick that is launched after this one and must return
    const u32 sv_base = views_of_tick(sched, p.tick);   // what this kernel's CTAs read when they started (nobody else writes these words)
    sched[SCHED_VIEWS_OLD] = sv_base; sched[SCHED_VIEWS_NEW] = sched[SCHED_VIEWS_NEXT] | sv_next; sched[SCHED_VIEWS_FROM] = p.tick + 1; sched[SCHED_VIEWS_NEXT] = 0;   // the views with business in the next tick (kernels that follow in this tick — anti-entropy, drain — add to it)
  }
  if (p.snd.world > 1 && p.fuse_publish) {
    // every CTA fenced its peer-window stores (system scope) before it took its ticket; this one saw all tickets
    __syncthreads();
    __threadfence();
    publish_to_peer(threadIdx.x, p.snd.world, p.snd.rank, p.xpar, p.stamp, p.loopback, p.peer_ctrl, p.snd.send_count, row, sched);
  }
}

// Persistent CTAs; each owns a contiguous range of 256-node tiles.  A tile is processed only if it is
// "hot": somebody delivered into it during the previous tick, it holds a node that stays awake (queued transmits,
// probe duty), a host operation targets it, or a suspicion timer of one of its nodes has come due — otherwise not a
// single byte of it is touched.
template <bool TRACE, int FMAX, bool SHARDED, bool R1, int MB, bool PASS = false>
__global__ void __launch_bounds__(BLOCK, MB) tick_kernel(const __grid_constant__ TickParams p) {
  __shared__ u8 hot_s[MAX_TILES_PER_CTA];
  __shared__ u64 red[8][BLOCK / 32];
  __shared__ int dsusp_s;                                  // net change of the number of Suspect views at up nodes, this CTA
  __shared__ __align__(16) unsigned char xs_mem[SHARDED ? sizeof(XStage) : 16];
  XStage* xs = reinterpret_cast<XStage*>(xs_mem);
  if (gate_closed(p.gate, blockIdx.x == 0 && threadIdx.x == 0)) return;   // the run is over (uniform over the grid): this tick does not exist
  if (tick_is_idle(p.sched, p.tick, p.ev_begin, p.ev_end)) { if (PASS ? p.sv_slot == 0 : p.sv_mode != SV_SINGLE) write_idle_row<TRACE>(p); return; }   // nothing can happen in this tick (uniform)
  // Single-view ticks of multi-slot runs (tick_kernel.cuh, SV_*): the general kernel and the single-view kernel are both launched; the
  // set of views that can have business in this tick — known on the device since the end of the previous tick — decides which one runs.
  u32 sv_views = 0xffffffffu;
  bool work = true, carry_out = false;                     // PASS: this pass's view has business; so has a later pass's
  if (PASS) {
    const u32 views = (views_of_tick(p.sched, p.tick) | p.views_host) & ((1u << p.sv_R) - 1u);
    work = (views >> p.sv_slot) & 1u;
    carry_out = (views >> p.sv_slot) > 1u;
    if (work) SFS_PROBE(21);
    else if (p.sv_slot != 0 && p.sv_slot + 1u < p.sv_R) return;    // neither node work nor a duty of the first or the last pass
  } else if (p.sv_mode != SV_OFF) {
    // (the kernel of this tick that ran before this one, if any, has already published the NEXT tick's set: SCHED_VIEWS_FROM says since when it holds)
    const u32 views = (views_of_tick(p.sched, p.tick) | p.views_host) & ((1u << p.sv_R) - 1u);
    const bool single = views == (1u << p.sv_slot);        // exactly the one view the single-view launch was set up for
    if (p.sv_mode == SV_SINGLE) { if (!single) return; SFS_PROBE(21); }
    else if (p.sv_mode == SV_GENERAL && single) return;
    if (p.sv_mode == SV_CHECK && (single || p.snd.world == 1)) sv_views = views;   // checked where the single-view kernel or the passes would have run
  }
  if (threadIdx.x == 0) dsusp_s = 0;                       // ordered before its first use by the barrier after the tile scan
  Counters c = {};
  // What this launch loads: the inbox planes of the kinds in flight, and (below) whether every node is requested up front.  A pass decides
  // from its own view's traffic (view_kinds_prev, tick_kernel.cuh): a plane no sender of its view wrote is zero and stays unread.
  const u32* const kv = PASS ? p.view_kinds_prev : p.kinds_prev;
  const bool kL = kv[KIND_LEAVE] != 0, kJ = kv[KIND_JOIN] != 0, kM = kv[KIND_ML] != 0;
  const u64 pol_first = policy_evict_first(), pol_last = policy_evict_last();
  const int lane = threadIdx.x & 31;
  if (SHARDED && threadIdx.x < (BLOCK / 32) * MAX_WORLD) xs->cnt[threadIdx.x / MAX_WORLD][threadIdx.x % MAX_WORLD] = 0;
  bool wrote_remote = false;
  u32 resv = 0, rlen = 0;                                  // lane s: the entries this warp holds reserved in peer s's window (flush_xwarp)

  // Dense / sparse ticks (dense_tick, tick_kernel.cuh): kinds[3] of this tick's counters records the decision.
  const u32 prev_msgs = sent_messages(p.kinds_prev);
  const bool dense_now = dense_tick(prev_msgs, p.n_tiles);       // what this tick's sends will look like
  const bool all_hot = p.force_all || p.kinds_prev[3] != 0;      // the previous tick was dense (or skipping is off)
  const bool mark = !dense_now;
  const u32 own_msgs = PASS ? sent_messages(kv) : prev_msgs;
  const bool saturated = own_msgs >= (p.n_local >> 1);           // most nodes have mail: request record + node word up front
  if (dense_now && blockIdx.x == 0 && threadIdx.x == 0) p.kinds_cur[3] = 1;
  if (PASS && work && threadIdx.x == 0) {                        // coverage of the host build: decisions the whole-tick counters would have taken otherwise
    if (kv == p.kinds_prev) SFS_PROBE(23);                       // whole-tick fallback (an earlier writer of the inbox was not a pass)
    if (!saturated && prev_msgs >= (p.n_local >> 1) && p.compact) SFS_PROBE(24);   // compacted walk in a tick another view saturates
    if ((!kL && p.kinds_prev[KIND_LEAVE]) || (!kJ && p.kinds_prev[KIND_JOIN]) || (!kM && p.kinds_prev[KIND_ML])) SFS_PROBE(25);   // a plane of a kind in flight elsewhere, not read
  }

  const u32 tile0 = blockIdx.x * p.tiles_per_cta;
  const u32 ntile = tile0 < p.n_tiles ? min(p.tiles_per_cta, p.n_tiles - tile0) : 0;
  if (SHARDED && saturated && ntile && (u32)lane < p.snd.world && (u32)lane != p.snd.rank) { resv = atomicAdd(p.snd.send_count + lane, XW_FLUSH); rlen = XW_FLUSH; }   // every warp will send to every peer
  if (PASS && p.sv_slot != 0) tile_decisions(p, hot_s, tile0, ntile, p.sv_slot + 1u == p.sv_R, work); else scan_tiles(p, hot_s, tile0, ntile, all_hot, PASS);
  __syncthreads();
  if (PASS && !work && p.sv_slot + 1u < p.sv_R) return;   // the first pass without business has made the tiles' decisions
  // Unsaturated ticks (ramp-up and tail of a dissemination: a few per cent of the nodes have anything to do, spread
  // one or two per warp): a tile-by-tile walk pays one chain of dependent round trips (state → row → peers) per TILE
  // for a handful of active lanes.  Instead the CTA scans GROUP hot tiles at once — the 13 "anything to do?" bytes
  // of every node, all loads in flight together — compacts the active nodes into a shared-memory list and runs the
  // node logic on dense blocks of 256 list entries: one chain per 256 ACTIVE nodes.  Nodes are independent within a
  // tick and every cross-node effect is a commutative reduction, so the visiting order changes nothing.
  constexpr u32 GROUP = SHARDED ? 4 : 8;
  __shared__ uint4 act_s[GROUP * BLOCK];                   // x: tile-in-group << 8 | lane, busy << 16, any << 24; y, z, w: inbox words
  __shared__ u32 act_n;
  __shared__ u8 pend_s[GROUP];
  __shared__ u16 gt_s[GROUP];
  const bool compact = !TRACE && !saturated && !p.reap_now && p.compact;
  if (compact) {
    u32 i = 0;
    while (i < ntile) {
      u32 ng = 0;                                          // the next GROUP hot tiles of this CTA (every thread walks the same flags)
      while (i < ntile && ng < GROUP) { if (hot_s[i]) { if (threadIdx.x == 0) gt_s[ng] = (u16)i; ++ng; } ++i; }
      if (!ng) break;
      if (threadIdx.x == 0) act_n = 0;
      if (threadIdx.x < GROUP) pend_s[threadIdx.x] = 0;
      __syncthreads();
      Pre pr[GROUP];
#pragma unroll
      for (u32 g = 0; g < GROUP; ++g) {
        pr[g] = Pre{};
        if (g < ng) {
          const u32 vn = ((tile0 + gt_s[g]) << TILE_SHIFT) + threadIdx.x;
          if (vn < p.n_local) pr[g] = prefetch_node<R1, PASS>(p, vn, kL, kJ, kM, pol_first, PASS && (hot_s[gt_s[g]] & 2u) != 0);   // (a node's own deadline is read below, in due tiles only: eight more live registers otherwise)
        }
      }
#pragma unroll
      for (u32 g = 0; g < GROUP; ++g) {
        const bool due_g = g < ng && (hot_s[gt_s[g]] & 2u) != 0;
        Pre prg = pr[g];
        if (due_g && (prg.busy & BUSY_TIMER)) prg.nd = ld_node_due(p.node_due + ((tile0 + gt_s[g]) << TILE_SHIFT) + threadIdx.x, pol_first);
        const bool act = g < ng && node_active<PASS>(p, prg, due_g);   // lanes past n_local hold an empty Pre
        if (due_g) {                                         // (warp-uniform) nodes whose own timers run later hand their deadline back to the wheel
          const u32 wm = warp_min(act ? NO_DEADLINE : sleeping_deadline(prg, true));
          if (lane == 0 && wm != NO_DEADLINE) atomicMin(p.tile_due + tile0 + gt_s[g], wm);
          if (!act && (prg.busy & BUSY_TIMER)) SFS_PROBE(20);
        }
        const u32 bal = __ballot_sync(0xffffffffu, act);
        if (bal) {
          u32 base = 0;
          if (lane == 0) base = atomicAdd(&act_n, (u32)__popc(bal));
          base = __shfl_sync(0xffffffffu, base, 0);
          if (act) act_s[base + (u32)__popc(bal & ((1u << lane) - 1u))] =
              make_uint4((g << 8) | threadIdx.x | (pr[g].busy << 16) | ((pr[g].any ? 1u : 0u) << 24), pr[g].mL, pr[g].mJ, pr[g].mM);
        }
      }
      __syncthreads();
      const u32 na = act_n;
      if (threadIdx.x == 0) { SFS_PROBE(0); if (ng > 1) SFS_PROBE(1); if (na > BLOCK) SFS_PROBE(2); }   // groups, multi-tile groups, multi-pass groups
      for (u32 b0 = 0; b0 < na; b0 += BLOCK) {
        const u32 e = b0 + threadIdx.x;
        if (e < na) {
          const uint4 a = act_s[e];
          const u32 g = (a.x >> 8) & 0xffu;
          const u32 ti = gt_s[g];
          const u32 vl = ((tile0 + ti) << TILE_SHIFT) + (a.x & 0xffu);
          Pre pre;
          if (R1) {
            pre.busy = (a.x >> 16) & 0xffu; pre.any = (a.x >> 24) & 1u; pre.mL = a.y; pre.mJ = a.z; pre.mM = a.w; pre.keep = 0;
            pre.nd = NO_DEADLINE;
            pre.qw = ld_qword(p.qword + vl, pol_first);           // not carried through the list: issued here, in flight with the state loads
            pre.mailmask = pre.any ? 1u : 0u; pre.qmask = pre.qw ? 1u : 0u;
            SFS_COUNT(6, 4);
          } else {
            pre = prefetch_node<R1, PASS>(p, vl, kL, kJ, kM, pol_first, (hot_s[ti] & 2u) != 0);   // per-view masks are not carried through the list: the few active nodes read them again
          }
          u32 mind = NO_DEADLINE, fv_unused = 0;
          int dsusp = 0;
          const bool pend = process_node<TRACE, FMAX, SHARDED, R1, false, PASS>(p, StageView{}, xs, vl, pre, kL, kJ, kM, mark, false, (hot_s[ti] & 2u) != 0, pol_first, pol_last, c, mind, dsusp, Ahead<FMAX>{}, fv_unused, sv_views, carry_out);
          if (mark && pend) pend_s[g] = 1;
          if (mind != NO_DEADLINE) atomicMin(p.tile_due + tile0 + ti, mind);      // the list mixes tiles: per-lane registration (few active nodes)
          if (dsusp) atomicAdd(&dsusp_s, dsusp);
        }
        if (SHARDED) wrote_remote |= flush_xwarp(p, xs, false, resv, rlen);
      }
      __syncthreads();
      if (mark && threadIdx.x < ng && pend_s[threadIdx.x]) p.hot_wr[tile0 + gt_s[threadIdx.x]] = 1;
      __syncthreads();                                     // gt_s / act_s are rewritten by the next group
    }
  } else {
  // Walk the hot tiles of this CTA.  The 13 "is there anything to do" bytes of the NEXT hot tile (busy byte, inbox
  // words) are requested before the current tile is processed, so an idle tile costs no exposed round trip.
  // Multi-slot runs, saturated ticks: node word, peers' ids and the probable first view's record travel one tile ahead too (Ahead).
  const bool ahead_on = !R1 && p.udeg != 0 && (p.ahead == 2u || (p.ahead == 1u && saturated));
  u32 first_view = 0;                                      // the first view this thread visited in its last tile
  auto prefetch_tile = [&](u32 ti) -> Pre {
    const u32 vn = ((tile0 + ti) << TILE_SHIFT) + threadIdx.x;
    return vn < p.n_local ? prefetch_node<R1, PASS>(p, vn, kL, kJ, kM, pol_first, (hot_s[ti] & 2u) != 0, first_view) : Pre{};
  };
  auto ahead_tile = [&](u32 ti, u32 keep) -> Ahead<FMAX> {
    Ahead<FMAX> a = {};
    const u32 vn = ((tile0 + ti) << TILE_SHIFT) + threadIdx.x;
    if (!R1 && ahead_on && vn < p.n_local) {
      a.ns = ld_u64_stream(p.node_state + vn, pol_first);
      a.rec = ld_rec256(p.rec + 2 * ((size_t)keep * p.stride + vn), pol_first);
      pick_issue<FMAX, false>(p, StageView{}, p.first + vn, vn * p.udeg, p.udeg, pol_first, a.cand);
      a.valid = 1;
      SFS_PROBE(19);
    }
    return a;
  };
  u32 i = 0;
  while (i < ntile && !hot_s[i]) ++i;
  Pre pre_next = {};
  Ahead<FMAX> ah_next = {};
  if (i < ntile) { pre_next = prefetch_tile(i); ah_next = ahead_tile(i, pre_next.keep); }
  while (i < ntile) {
    const Pre pre = pre_next;
    const Ahead<FMAX> ah = ah_next;
    u32 j = i + 1;
    while (j < ntile && !hot_s[j]) ++j;
    if (j < ntile) { pre_next = prefetch_tile(j); ah_next = ahead_tile(j, pre_next.keep); }
    const u32 vl = ((tile0 + i) << TILE_SHIFT) + threadIdx.x;
    bool pend = false;
    u32 mind = NO_DEADLINE;
    int dsusp = 0;
    if (vl < p.n_local) pend = process_node<TRACE, FMAX, SHARDED, R1, false, PASS>(p, StageView{}, xs, vl, pre, kL, kJ, kM, mark, saturated, (hot_s[i] & 2u) != 0, pol_first, pol_last, c, mind, dsusp, ah, first_view, sv_views, carry_out);
    if (mark && __any_sync(0xffffffffu, pend) && lane == 0) p.hot_wr[tile0 + i] = 1;
    note_timers(p, tile0 + i, mind, dsusp, &dsusp_s);
    if (SHARDED) wrote_remote |= flush_xwarp(p, xs, false, resv, rlen);
    i = j;
  }
  }
  if (SHARDED) {
    wrote_remote |= flush_xwarp(p, xs, true, resv, rlen);
    if (wrote_remote) __threadfence_system();            // peer-window stores are performed before the publish kernel raises the flags
  }
  __syncthreads();
  finish_tick<TRACE, R1, PASS>(p, c, red, dsusp_s);
}

#ifndef SERFSIM_EMU   // the TMA pipeline is device-only (bulk copies, mbarriers); the host build of tests/emu uses the direct-load kernel
// The same tick for single-slot runs with the whole working set of a tile staged through TMA: one elected
// thread bulk-copies the tile's records (8 KB), node words (2 KB), live inbox planes (1 KB each), row offsets
// (1 KB) and CSR span (the tile's neighbour lists, 16 KB at out-degree 16) into shared memory, one tile ahead
// of the 256 consumers (2 stages, mbarrier transaction counts).  The node logic then runs out of shared memory;
// only the RED.MAX sends, the record write-back and the inbox clears touch global memory from the LSU.
template <bool TRACE, int FMAX, bool SHARDED, bool BARSYNC>
__global__ void __launch_bounds__(BLOCK, 3) tick_kernel_tma(const __grid_constant__ TickParams p) {
  extern __shared__ __align__(128) unsigned char stage_mem[];
  __shared__ u8 hot_s[MAX_TILES_PER_CTA];
  __shared__ u16 hot_list[MAX_TILES_PER_CTA];
  __shared__ u32 n_hot_s;
  __shared__ u64 red[8][BLOCK / 32];
  __shared__ __align__(8) u64 full_bar[2], empty_bar[2];
  __shared__ u32 col_base_s[2], col_ok_s[2];
  __shared__ int dsusp_s;
  if (gate_closed(p.gate, blockIdx.x == 0 && threadIdx.x == 0)) return;
  if (tick_is_idle(p.sched, p.tick, p.ev_begin, p.ev_end)) { write_idle_row<TRACE>(p); return; }
  Counters c = {};
  const bool kL = p.kinds_prev[KIND_LEAVE] != 0, kJ = p.kinds_prev[KIND_JOIN] != 0, kM = p.kinds_prev[KIND_ML] != 0;
  const u64 pol_first = policy_evict_first(), pol_last = policy_evict_last();
  const int lane = threadIdx.x & 31;

  const bool dense_now = dense_tick(sent_messages(p.kinds_prev), p.n_tiles);
  const bool all_hot = p.force_all || p.kinds_prev[3] != 0;
  const bool mark = !dense_now;
  if (dense_now && blockIdx.x == 0 && threadIdx.x == 0) p.kinds_cur[3] = 1;

  const u32 tile0 = blockIdx.x * p.tiles_per_cta;
  const u32 ntile = tile0 < p.n_tiles ? min(p.tiles_per_cta, p.n_tiles - tile0) : 0;
  scan_tiles(p, hot_s, tile0, ntile, all_hot);
  if (threadIdx.x == 0) {
    dsusp_s = 0;
    mbar_init(&full_bar[0], 1); mbar_init(&full_bar[1], 1);
    mbar_init(&empty_bar[0], BLOCK / 32); mbar_init(&empty_bar[1], BLOCK / 32);     // one arrival per consumer warp
    fence_proxy_async();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    u32 n = 0;
    for (u32 i = 0; i < ntile; ++i) if (hot_s[i]) hot_list[n++] = (u16)i;
    n_hot_s = n;
  }
  __syncthreads();
  const u32 n_hot = n_hot_s;
  const u32 stage_bytes = ST_COL + p.stage_col_bytes;

  // producer: bulk-copy tile `j` of the hot list into stage j&1
  auto issue = [&](u32 j) {
    const u32 st = j & 1;
    unsigned char* base = stage_mem + (size_t)st * stage_bytes;
    const u32 tile = tile0 + hot_list[j];
    const u32 v0 = tile << TILE_SHIFT;
    const u32 e0 = __ldg(p.row_ptr + v0) & ~3u;
    const u32 e1 = (__ldg(p.row_ptr + min(v0 + BLOCK, p.n_local)) + 3u) & ~3u;
    const u32 col_bytes = (e1 - e0) * 4u;
    const bool col_ok = col_bytes != 0 && col_bytes <= p.stage_col_bytes;
    col_base_s[st] = e0; col_ok_s[st] = col_ok ? 1u : 0u;
    const u32 tx = 8192u + 2048u + RP_BYTES + (kL ? 1024u : 0u) + (kJ ? 1024u : 0u) + (kM ? 1024u : 0u) + (col_ok ? col_bytes : 0u);
    fence_proxy_async();                                   // earlier generic reads of this stage precede the async writes
    mbar_arrive_expect_tx(&full_bar[st], tx);
    bulk_g2s(base + ST_REC, p.rec + 2 * (size_t)v0, 8192u, &full_bar[st], pol_first);
    bulk_g2s(base + ST_NODE, p.node_state + v0, 2048u, &full_bar[st], pol_first);
    bulk_g2s(base + ST_RP, p.row_ptr + v0, RP_BYTES, &full_bar[st], pol_first);
    if (kL) bulk_g2s(base + ST_INL, p.inbox_rd + (size_t)KIND_LEAVE * p.stride + v0, 1024u, &full_bar[st], pol_first);
    if (kJ) bulk_g2s(base + ST_INJ, p.inbox_rd + (size_t)KIND_JOIN * p.stride + v0, 1024u, &full_bar[st], pol_first);
    if (kM) bulk_g2s(base + ST_INM, p.inbox_rd + (size_t)KIND_ML * p.stride + v0, 1024u, &full_bar[st], pol_first);
    if (col_ok) bulk_g2s(base + ST_COL, p.col + e0, col_bytes, &full_bar[st], pol_first);
  };

  // No CTA-wide barrier in the loop: a warp that finishes a tile arrives on the stage's `empty` barrier and
  // moves on; only the producer (thread 0) waits for all eight warps to release a stage before refilling it.
  if (threadIdx.x == 0 && n_hot) issue(0);
  for (u32 j = 0; j < n_hot; ++j) {
    if (threadIdx.x == 0 && j + 1 < n_hot) {
      if (!BARSYNC && j >= 1) mbar_wait(&empty_bar[(j + 1) & 1], ((j - 1) >> 1) & 1);   // tile j-1 (same stage) fully consumed
      issue(j + 1);
    }
    const u32 st = j & 1;
    mbar_wait(&full_bar[st], (j >> 1) & 1);
    unsigned char* base = stage_mem + (size_t)st * stage_bytes;
    StageView sv;
    sv.rec = reinterpret_cast<const Words*>(base + ST_REC); sv.node = reinterpret_cast<const u64*>(base + ST_NODE);
    sv.inL = reinterpret_cast<const u32*>(base + ST_INL); sv.inJ = reinterpret_cast<const u32*>(base + ST_INJ); sv.inM = reinterpret_cast<const u32*>(base + ST_INM);
    sv.rowptr = reinterpret_cast<const u32*>(base + ST_RP); sv.col = reinterpret_cast<const u32*>(base + ST_COL);
    sv.col_base = col_base_s[st]; sv.col_staged = col_ok_s[st] != 0;
    const u32 ti = hot_list[j];
    const u32 vl = ((tile0 + ti) << TILE_SHIFT) + threadIdx.x;
    bool pend = false;
    u32 mind = NO_DEADLINE;
    int dsusp = 0;
    if (vl < p.n_local) {
      Pre pre = {};
      pre.busy = p.busy[vl];
      pre.qw = p.qword[vl];          // 4 B per node, read directly (not worth a sixth bulk copy per stage)
      pre.nd = NO_DEADLINE;
      u32 fv_unused = 0;
      pend = process_node<TRACE, FMAX, false, true, true>(p, sv, nullptr, vl, pre, kL, kJ, kM, mark, true, (hot_s[ti] & 2u) != 0, pol_first, pol_last, c, mind, dsusp, Ahead<FMAX>{}, fv_unused);
    }
    if (mark && __any_sync(0xffffffffu, pend) && lane == 0) p.hot_wr[tile0 + ti] = 1;
    note_timers(p, tile0 + ti, mind, dsusp, &dsusp_s);
    if (BARSYNC) __syncthreads();
    else { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[st]); }     // this warp is done reading stage `st`
  }

  __syncthreads();
  finish_tick<TRACE, true>(p, c, red, dsusp_s);
}
#endif

// Anti-entropy round — memberlist push-pull + SerfDelegate::merge_remote_state (serf/delegate.rs:386-554; "next"
// row 1 of SURVEY §8f).  Runs after the tick kernel every push_pull_interval ticks on a SNAPSHOT of the end-of-tick
// state: each up node pulls the state of one random neighbour and merges it — clock witness(ltime−1), per subject
// the memberlist state (alive → aliveNode, suspect/dead → suspectNode{from = self}, left → deadNode{from = node}),
// then serf's view (Left member → leave intent at status_ltime+1, any other → join intent at status_ltime) with the
// handlers' results discarded: nothing is re-queued (delegate.rs:495-523).  A node writes only its own records.
template <bool TRACE>
__global__ void __launch_bounds__(BLOCK) pushpull_kernel(const __grid_constant__ TickParams p, const uint4* __restrict__ snap_rec, const u64* __restrict__ snap_node) {
  if (p.gate.ctl && p.gate.ctl[0]) return;
  // a round can queue transmits and start timers after the tick kernel has decided how long the cluster may sleep: take the decision back
  if (blockIdx.x == 0 && threadIdx.x == 0) { p.sched[SCHED_IDLE_UNTIL] = 0; if (p.host_idle_until) *p.host_idle_until = 0; }
  long long d_changed = 0, d_pending = 0, d_susp = 0;
  u64 d_hash = 0;
  u32 d_views = 0;                                         // views left with queued transmits: they have business in the next tick
  for (u32 vl = blockIdx.x * BLOCK + threadIdx.x; vl < p.n_local; vl += gridDim.x * BLOCK) {
    const u32 v = p.first + vl;
    const u64 ns = snap_node[vl];
    if (!nw_up(ns)) continue;
    const u32 row0 = p.row_ptr[vl], deg = p.row_ptr[vl + 1] - row0;
    if (!deg) continue;
    const u32 u = p.col[row0 + neighbour_slot(p.tick, v, DOMAIN_PUSHPULL, p.seed_lo, p.seed_hi, deg)];
    if (u == v) continue;
    // the partner may live in another shard: its rank's snapshot is read through the peer mapping (the host
    // separates "every rank has taken its snapshot" and "every rank has finished reading" with barriers)
    u32 ul = u - p.first;
    const u64* part_node = snap_node;
    const uint4* part_rec = snap_rec;
    u32 part_stride = p.stride;
    u32 shard = 0;
    if (p.snd.world > 1) {
      const ShardIdx t = shard_of(u, p.snd.shard_size, p.snd.shard_inv);
      shard = t.shard; ul = t.local;
      part_node = p.snap_node_peer[shard]; part_rec = p.snap_rec_peer[shard];
      part_stride = shard_span(shard, p.snd.shard_size, p.n_global).stride;
    }
    const u64 nu = part_node[ul];
    if (!nw_up(nu)) continue;
    u32 clock = nw_clock(ns);
    const u32 sstate = nw_sstate(ns);
    const u32 cu = nw_clock(nu);
    if (cu > 0) witness(clock, cu - 1);
    bool awake = false, has_timer = false;
    u32 mind = NO_DEADLINE;
    const u32 wmask = p.watch[vl];
    for (u32 s = 0; s < p.R; ++s) {
      const size_t iv = (size_t)s * p.stride + vl, iu = (size_t)s * part_stride + ul;
      Words w0 = load_rec(p.rec, iv);
      const u32 q0 = p.qword[iv];
      merge_queue_word(w0, q0);
      Rec r, q;
      unpack(w0, r);
      unpack(load_rec(part_rec, iu), q);
      const bool self = (p.subj[s] == v);
      const bool watching = view_watching(wmask != 0, p.probe_every, p.down_mask, s, self, wmask);
      const bool was = view_pending(r, watching) || r.mlstate == ML_SUSPECT;
      if (q.flags & 1) {
        if (q.mlstate == ML_ALIVE) ml_alive(r, q.inc, self, p.rules.limit);
        else if (q.mlstate == ML_LEFT) ml_dead(r, q.inc, true, p.tick, self, p.rules.limit);
        else ml_suspect(r, q.inc, from_bucket(v), p.tick, self, p.rules);
        bool refute = false;
        if (q.status == ST_LEFT) { witness(clock, q.st + 1); leave_intent(r, q.st + 1, false, self, sstate, refute, p.rules.limit, false); }
        else { witness(clock, q.st); join_intent(r, q.st, p.rules.limit, false); }
        if (refute) refute_leave(r, clock, p.rules.limit);
        stamp_intent(r, w0, p.tick);
      }
      Words w1;
      pack(r, w1);
      const bool ch = differs(w1, w0);
      if (ch) {
        Words ws = w1;
        const u32 q1 = split_queue_word(ws);
        store_rec(p.rec, iv, ws);
        if (q1 != q0) p.qword[iv] = q1;
      }
      Words wt = w1;                                       // status_time creep is not a change
      wt.w[0] = w0.w[0];
      if (differs(wt, w0)) { d_changed++; SFS_PROBE(28); }
      if (TRACE && ch) d_hash += rec_hash((u64)s * p.n_global + v, w1) - rec_hash((u64)s * p.n_global + v, w0);
      d_pending += (view_pending(r, watching) || r.mlstate == ML_SUSPECT ? 1 : 0) - (was ? 1 : 0);
      d_susp += (r.mlstate == ML_SUSPECT ? 1 : 0) - (((w0.w[6] >> 8) & 3u) == ML_SUSPECT ? 1 : 0);     // the node is up: counted views
      awake |= view_awake(r, watching, [&] { return can_confirm(p.rules.k, r.mask, v); });
      if (r.mlstate == ML_SUSPECT && r.deadline != 0) { has_timer = true; mind = min(mind, r.deadline); }
      if (rec_queued(r)) d_views |= 1u << s;
      if (r.inc >= INC_LIMIT) *p.overflow = 1;
    }
    if (p.ue_table.n) {                                        // the partner's event clock and ring (a snapshot, like its records)
      const uint4 pw = (p.snd.world > 1 ? p.ue_snap_peer[shard] : p.ue_snap)[ul];
      const uint4 w0 = p.ue_state[vl];
      UeRec er;
      ue_unpack(w0, er);
      UeCounts ec = {};
      ue_replay(er, pw.x, pw.y & 0xffu, p.ue_ltime, p.ue_table, p.rules.limit, ec);
      const uint4 w1 = ue_pack(er);
      if ((w1.x ^ w0.x) | (w1.y ^ w0.y) | (w1.z ^ w0.z) | (w1.w ^ w0.w)) p.ue_state[vl] = w1;
      d_changed += ec.delivered;
      if (ec.delivered) atomicAdd((unsigned long long*)(p.ue_totals + 2), (unsigned long long)ec.delivered);
      if (ec.duplicates) atomicAdd((unsigned long long*)(p.ue_totals + 3), (unsigned long long)ec.duplicates);
      if (ec.too_old) atomicAdd((unsigned long long*)(p.ue_totals + 4), (unsigned long long)ec.too_old);
      if (TRACE) d_hash += ue_hash((u64)(p.R + 1) * p.n_global + v, w1) - ue_hash((u64)(p.R + 1) * p.n_global + v, w0);
      if (er.clock >= LTIME_LIMIT) *p.overflow = 1;
    }
    const u64 ns2 = node_word(clock, nw_up(ns), sstate);
    if (ns2 != ns) {
      p.node_state[vl] = ns2;
      if (TRACE) d_hash += node_hash((u64)p.R * p.n_global + v, ns2) - node_hash((u64)p.R * p.n_global + v, ns);
    }
    if (clock >= LTIME_LIMIT) *p.overflow = 1;
    // every view of the node was visited: its busy byte is exact
    p.busy[vl] = (u8)((awake ? BUSY_AWAKE : 0u) | (wmask ? BUSY_WATCH : 0u) | (has_timer ? BUSY_TIMER : 0u));
    if (awake) p.hot_wr[vl >> TILE_SHIFT] = 1;
    if (has_timer) { atomicMin(p.tile_due + (vl >> TILE_SHIFT), mind); p.node_due[vl] = mind; }
  }
  const u64 c = warp_sum64((u64)d_changed), q = warp_sum64((u64)d_pending), ds = warp_sum64((u64)d_susp), h = TRACE ? warp_sum64(d_hash) : 0;
  d_views = __reduce_or_sync(0xffffffffu, d_views);
  if ((threadIdx.x & 31) == 0) {
    if (d_views) atomicOr(p.sched + SCHED_VIEWS_NEW, d_views);
    if (c) atomicAdd((unsigned long long*)(p.row + ROW_CHANGED), (unsigned long long)c);
    if (q) atomicAdd((unsigned long long*)(p.row + ROW_PENDING), (unsigned long long)q);
    if (ds) atomicAdd(reinterpret_cast<unsigned long long*>(p.sched + SCHED_SUSPECTS), (unsigned long long)ds);
    if (TRACE && h) atomicAdd((unsigned long long*)(p.row + ROW_HASH), (unsigned long long)h);
  }
}

// After the tick kernel: publish, to every peer, how many entries this rank wrote into its window, then raise
// the peer's flag for this exchange (system-scope release).  One warp.
__global__ void publish_kernel(const __grid_constant__ PublishParams p) {
  if (p.gate && *p.gate) return;
  publish_to_peer(threadIdx.x, p.world, p.rank, p.xpar, p.stamp, p.loopback, p.peer_ctrl, p.send_count, p.row, p.sched);
}

// Fold the cross-shard windows into the inbox.  Waits (system-scope acquire) until every peer has raised
// this exchange's flag — the peers' publish kernels precede their own drains in stream order, so the wait
// cannot deadlock — then reduces the entries exactly like local deliveries.
__global__ void __launch_bounds__(BLOCK) drain_kernel(const __grid_constant__ DrainParams p) {
  if (p.gate && *p.gate) return;
  if (threadIdx.x < p.world && threadIdx.x != p.rank) {
    u32 f;
    do { f = ld_acquire_sys(p.flags + threadIdx.x); } while (f != p.stamp);
  }
  __syncthreads();
  // global trace row of this tick: my counters + the rows the peers published with their flags (acquired above)
  if (blockIdx.x == 0 && threadIdx.x < ROW_FIELDS) {
    u64 s = p.my_row[threadIdx.x];
    for (u32 src = 0; src < p.world; ++src) if (src != p.rank) s += __ldcg(&p.sums[src][threadIdx.x]);
    p.grow[threadIdx.x] = s;
  }
  // The ranks' scheduler verdicts: the cluster sleeps iff every rank is quiet, until the earliest of their deadlines.  Every rank
  // computes the same value from the same published words and hands it to its HOST only (mapped memory): in sharded runs the
  // device never skips a launched tick — a skipped exchange would let a fast rank reuse a window parity its peer is still
  // draining — the hosts simply do not launch the ticks the cluster sleeps through (serfsim_run_until_converged), all alike.
  if (blockIdx.x == 0 && threadIdx.x == 0 && p.sched) {
    bool quiet = p.sleep_on && p.sched[SCHED_LOCAL_QUIET] != 0;
    u32 until = p.sched[SCHED_LOCAL_UNTIL];
    for (u32 src = 0; src < p.world; ++src) {
      if (src == p.rank) continue;
      quiet = quiet && __ldcg(&p.sums[src][CTRL_QUIET]) != 0;
      until = min(until, (u32)__ldcg(&p.sums[src][CTRL_UNTIL]));
    }
    if (p.host_idle_until) *p.host_idle_until = quiet ? max(until, p.tick + 1) : p.tick + 1;
    u32 views = 0;                                        // views with business in the next tick: anywhere in the cluster (their mail crosses shards)
    for (u32 src = 0; src < p.world; ++src) if (src != p.rank) views |= (u32)__ldcg(&p.sums[src][CTRL_VIEWS]);
    if (views) atomicOr(p.sched_rw + SCHED_VIEWS_NEW, views);
  }
  // the tick kernel's dense / sparse decision of this tick: in a dense tick the next tick processes every
  // tile anyway, so per-entry tile marking (millions of byte stores onto a few thousand flags) is skipped
  const bool mark = !dense_tick(sent_messages(p.kinds_prev), p.n_tiles);
  u32 seen = 0;                                 // kinds this thread folded (bit per kind)
  for (u32 src = 0; src < p.world; ++src) {
    if (src == p.rank) continue;
    const u32 n = min(p.counts[src], p.win_cap);
    u64* w = win_segment(p.win_data, src, p.win_cap);
    for (u32 i = blockIdx.x * BLOCK + threadIdx.x; i < n; i += gridDim.x * BLOCK) {
      const u64 e = __ldcg(w + i);
      if (e == 0) continue;                          // padding of a partly filled block (a real entry has value + 1 > 0 in its high word)
      if (!p.byz_on) w[i] = 0;                       // consumed: the window reads as zeros when it is written next (injector triples are
                                                     // read by a neighbouring thread too: those runs clear the windows in a kernel of their own)
      const u32 val1 = win_val1(e), s = win_slot(e), kind = win_kind(e);
      u32 dl = win_dst(e);
      const bool byz = p.byz_on && (dl & BYZ_FLAG);
      if (byz) dl &= ~BYZ_FLAG;
      if (byz && kind == KIND_EXTRA && s == BYZ_ANNOT_SLOT) continue;           // third entry of a triple: read by the thread holding the first
      if (dl < p.n_local && s < p.R && kind < 3) {
        atomicMax(p.inbox_wr + ((size_t)(kind * p.R + s)) * p.stride + dl, val1);
        if (mark) p.hot_wr[dl >> TILE_SHIFT] = 1;
        seen |= 1u << kind;
        if (byz && kind < 2 && i + 2 < n) {                            // first entry of a triple: judge it against MY record, flag the sender in ITS shard
          const u64 e1 = __ldcg(w + i + 1), e2 = __ldcg(w + i + 2);
          const u32 src = win_val1(e2) - 1u;
          ByzEntries be{};
          be.serf_lt = kind == KIND_LEAVE ? leave_key_lt(val1 - 1u) : val1 - 1u; be.ml_inc = ml_key_inc(win_val1(e1) - 1u);
          if (nw_up(p.node_state[dl])) {
            Rec q;
            unpack(load_rec(p.rec, (size_t)s * p.stride + dl), q);
            if (byz_anomalous(q, be, p.byz_delta)) { const ShardIdx t = shard_of(src, p.shard_size, p.shard_inv); p.peer_anomaly[t.shard][t.local] = 1; }
          }
        }
      } else if (dl < p.n_local && kind == KIND_EXTRA && s < p.ue_n && val1) {   // user event s arrived: one bit, and the time its origin stamped
        atomicOr(p.ue_inbox_wr + dl, 1u << s);
        p.ue_ltime[s] = val1 - 1;                      // every copy carries the same value; this shard learns it no later than the event itself
      }
      else *p.overflow = 3;
    }
  }
  // received kinds count as "in flight" for the next tick's plane skipping; the received volume feeds its dense/sparse decision
  seen = __reduce_or_sync(0xffffffffu, seen);
  if ((threadIdx.x & 31) == 0 && seen) {
    for (u32 k = 0; k < 3; ++k) if ((seen >> k) & 1) atomicAdd(p.kinds_cur + k, 1u);
  }
}

// Rows of ticks the host did not launch because the cluster sleeps through them (serfsim_run_until_converged): what
// write_idle_row would have written.  rows = first of the n rows; the row before it belongs to the last executed / skipped tick.
__global__ void fill_idle_rows_kernel(u64* rows, u64* grow_rows, u32 n, const u32* sched, int trace) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u64* const row = rows + (size_t)i * ROW_FIELDS;
  row[ROW_PENDING] = *reinterpret_cast<const u64*>(sched + SCHED_SUSPECTS);
  if (trace) row[ROW_HASH] = *(rows - ROW_FIELDS + ROW_HASH);
  if (grow_rows) {                                         // sharded: the global rows repeat the global pending count / hash
    u64* const grow = grow_rows + (size_t)i * ROW_FIELDS;
    grow[ROW_PENDING] = *(grow_rows - ROW_FIELDS + ROW_PENDING);
    if (trace) grow[ROW_HASH] = *(grow_rows - ROW_FIELDS + ROW_HASH);
  }
}

// Injector runs: the drain kernel leaves its windows as they are (a triple is read by two threads); this clears what it consumed.
__global__ void __launch_bounds__(BLOCK) clear_windows_kernel(const __grid_constant__ DrainParams p) {
  if (p.gate && *p.gate) return;
  for (u32 src = 0; src < p.world; ++src) {
    if (src == p.rank) continue;
    const u32 n = min(p.counts[src], p.win_cap);
    u64* w = win_segment(p.win_data, src, p.win_cap);
    for (u32 i = blockIdx.x * BLOCK + threadIdx.x; i < n; i += gridDim.x * BLOCK) w[i] = 0;
  }
}

// watch[v]: bit s set iff subject s appears in node v's neighbour list — only such nodes can ever pick it as a probe
// target, so they alone evaluate the SWIM probe (and stay scheduled while it is down).
__global__ void compute_watch_kernel(const u32* __restrict__ row_ptr, const u32* __restrict__ col, const u32* __restrict__ subj, u32 R, u32 first, u32 n_local, u16* watch) {
  const u32 vl = blockIdx.x * blockDim.x + threadIdx.x;
  if (vl >= n_local) return;
  u32 m = 0;
  const u32 v = first + vl;
  for (u32 e = row_ptr[vl]; e < row_ptr[vl + 1]; ++e) {
    const u32 c = col[e];
    if (c == v) continue;
    for (u32 s = 0; s < R; ++s) m |= (c == subj[s]) ? (1u << s) : 0u;
  }
  watch[vl] = (u16)m;
}
__global__ void apply_watch_kernel(const u16* __restrict__ watch, u32 n_local, u8* busy, u8* hot_static) {
  const u32 vl = blockIdx.x * blockDim.x + threadIdx.x;
  if (vl >= n_local || watch[vl] == 0) return;
  busy[vl] |= BUSY_WATCH;
  hot_static[vl >> TILE_SHIFT] = 1;              // a watcher's tile is scheduled every tick (static flags: never consumed)
}

__global__ void init_state_kernel(uint4* rec, u64* node_state, u32 n_local, u32 stride, u32 R, u32 init_st, u32 init_clock) {
  const u32 vl = blockIdx.x * blockDim.x + threadIdx.x;
  if (vl >= n_local) return;
  Rec r = {};
  r.st = init_st; r.inc = 1; r.status = ST_ALIVE; r.mlstate = ML_ALIVE; r.flags = 1;
  Words x;
  pack(r, x);
  for (u32 s = 0; s < R; ++s) store_rec(rec, (size_t)s * stride + vl, x);
  node_state[vl] = node_word(init_clock, true, SS_ALIVE);
}

__global__ void mark_events_kernel(u8* busy, u8* hot_rd, const u32* ev_node, u32 ev_begin, u32 ev_end, u32 first, u32 n_local) {
  const u32 e = ev_begin + blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ev_end) return;
  const u32 vl = ev_node[e] - first;
  if (vl < n_local) {
    busy[vl] |= BUSY_OP;                           // one op per (node, tick): no two threads touch the same byte
    hot_rd[vl >> TILE_SHIFT] = 1;                  // the tile must run this tick
  }
}

__global__ void extract_kernel(const uint4* rec, const u64* node_state, u32 n_local, u32 stride, u32 slot, int what, void* out) {
  const u32 vl = blockIdx.x * blockDim.x + threadIdx.x;
  if (vl >= n_local) return;
  if (what == EXTRACT_CLOCK) { ((u64*)out)[vl] = nw_clock(node_state[vl]); return; }
  if (what == EXTRACT_CLOCK32) { ((u32*)out)[vl] = nw_clock(node_state[vl]); return; }
  Rec r;
  unpack(load_rec(rec, (size_t)slot * stride + vl), r);
  const bool known = r.flags & 1;
  switch (what) {
    case EXTRACT_STATUS: ((u8*)out)[vl] = known ? (u8)r.status : (u8)ST_NONE; break;
    case EXTRACT_STATUS_LTIME: ((u64*)out)[vl] = known ? r.st : 0; break;
    case EXTRACT_STATUS_LTIME32: ((u32*)out)[vl] = known ? r.st : 0; break;
    case EXTRACT_INC: ((u32*)out)[vl] = r.inc; break;
    case EXTRACT_ML: ((u8*)out)[vl] = (u8)r.mlstate; break;
  }
}

__global__ void compose_records_kernel(const uint4* rec, const u32* qword, u32 n_local, u32 stride, u32 slot, uint4* out) {
  const u32 vl = blockIdx.x * blockDim.x + threadIdx.x;
  if (vl >= n_local) return;
  const size_t idx = (size_t)slot * stride + vl;
  Words x = load_rec(rec, idx);
  merge_queue_word(x, qword[idx]);
  store_rec(out, vl, x);
}

__global__ void __launch_bounds__(BLOCK) state_hash_kernel(const uint4* rec, const u32* qword, const u64* node_state, u32 n_local, u32 stride, u32 first, u32 n_global, u32 R, u64* out) {
  u64 h = 0;
  for (u32 vl = blockIdx.x * BLOCK + threadIdx.x; vl < n_local; vl += gridDim.x * BLOCK) {
    for (u32 s = 0; s < R; ++s) {
      const size_t idx = (size_t)s * stride + vl;
      Words x = load_rec(rec, idx);
      merge_queue_word(x, qword[idx]);
      h += rec_hash((u64)s * n_global + first + vl, x);
    }
    h += node_hash((u64)R * n_global + first + vl, node_state[vl]);
  }
  h = warp_sum64(h);
  if ((threadIdx.x & 31) == 0 && h) atomicAdd((unsigned long long*)out, (unsigned long long)h);
}

// out[0] = max clock, out[1] = queued intents, out[2+2s] = min key, out[3+2s] = max key of slot s over
// up nodes other than the subject (agreement check for Stats / convergence studies).
__global__ void __launch_bounds__(BLOCK) summary_kernel(const uint4* rec, const u32* qword, const u64* node_state, u32 n_local, u32 stride, u32 first, u32 R, const u32* subj, u64* out) {
  u64 maxclock = 0, queued = 0;
  for (u32 s = 0; s < R; ++s) {
    u64 kmin = ~0ull, kmax = 0;
    const u32 sid = subj[s];
    for (u32 vl = blockIdx.x * BLOCK + threadIdx.x; vl < n_local; vl += gridDim.x * BLOCK) {
      const u64 ns = node_state[vl];
      if (s == 0) maxclock = max(maxclock, (u64)nw_clock(ns));
      const size_t idx = (size_t)s * stride + vl;
      Rec r;
      unpack(load_rec(rec, idx), r);
      { const u32 q = qword[idx]; queued += ((q & 0xffu) ? 1 : 0) + (((q >> 8) & 0xffu) ? 1 : 0); }
      if (nw_up(ns) && sid != first + vl) {
        const bool known = r.flags & 1;
        const u64 key = (((u64)r.st << 32) ^ ((u64)r.inc << 8) ^ ((u64)(known ? r.status : 0) << 4) ^ r.mlstate ^ ((u64)known << 63));
        kmin = min(kmin, key); kmax = max(kmax, key);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, o));
      kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, o));
    }
    if ((threadIdx.x & 31) == 0) {
      atomicMin((unsigned long long*)(out + 2 + 2 * s), (unsigned long long)kmin);
      atomicMax((unsigned long long*)(out + 3 + 2 * s), (unsigned long long)kmax);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) maxclock = max(maxclock, __shfl_xor_sync(0xffffffffu, maxclock, o));
  queued = warp_sum64(queued);
  if ((threadIdx.x & 31) == 0) {
    atomicMax((unsigned long long*)out, (unsigned long long)maxclock);
    if (queued) atomicAdd((unsigned long long*)(out + 1), (unsigned long long)queued);
  }
}

}  // namespace

int tick_ctas_per_sm_r1() { return SFS_MB_R1; }
int tick_ctas_per_sm_r1s() { return SFS_MB_R1S; }
int tick_ctas_per_sm_rn() { return SFS_MB_RN; }
int tick_grid_size(u32 n_local, int ctas_per_sm, int sms, int gridmul) {
  const u32 tiles = plane_stride(n_local) >> TILE_SHIFT;
  u32 grid = (u32)sms * (u32)ctas_per_sm * (u32)gridmul;    // persistent: SM count × resident CTAs × 2 (two waves for balance)
  if (tiles < grid) grid = tiles ? tiles : 1;
  while ((tiles + grid - 1) / grid > MAX_TILES_PER_CTA) grid += (u32)sms * (u32)ctas_per_sm;
  return (int)grid;
}

#ifndef SERFSIM_EMU
template <bool TRACE, int FMAX, bool SHARDED>
static void launch_tick_tma(const TickParams& p, int grid, bool barsync, cudaStream_t st) {
  const size_t smem = 2 * (size_t)(ST_COL + p.stage_col_bytes);
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(tick_kernel_tma<TRACE, FMAX, SHARDED, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(tick_kernel_tma<TRACE, FMAX, SHARDED, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    configured = true;
  }
  if (barsync) SFS_LAUNCH(grid, BLOCK, smem, st, tick_kernel_tma<TRACE, FMAX, SHARDED, true>)(p);
  else SFS_LAUNCH(grid, BLOCK, smem, st, tick_kernel_tma<TRACE, FMAX, SHARDED, false>)(p);
}
#endif

template <bool TRACE, int FMAX>
static void launch_tick_v(const TickParams& p, int grid, int ctas_per_sm, bool tma_sync, cudaStream_t st) {
  const bool sharded = p.snd.world > 1, r1 = p.R == 1;
#ifndef SERFSIM_EMU
  if (r1 && p.stage_col_bytes && !sharded) { // single-slot, single-GPU run whose tiles fit a shared-memory stage: TMA pipeline
    launch_tick_tma<TRACE, FMAX, false>(p, grid, tma_sync, st);
    return;
  }
#endif
  if (sharded) { if (r1) SFS_LAUNCH(grid, BLOCK, 0, st, tick_kernel<TRACE, FMAX, true, true, SFS_MB_R1S>)(p); else SFS_LAUNCH(grid, BLOCK, 0, st, tick_kernel<TRACE, FMAX, true, false, SFS_MB_RN>)(p); }
  else if (r1) { if (ctas_per_sm == 5) SFS_LAUNCH(grid, BLOCK, 0, st, tick_kernel<TRACE, FMAX, false, true, 5>)(p); else SFS_LAUNCH(grid, BLOCK, 0, st, tick_kernel<TRACE, FMAX, false, true, SFS_MB_R1>)(p); }
  else SFS_LAUNCH(grid, BLOCK, 0, st, tick_kernel<TRACE, FMAX, false, false, SFS_MB_RN>)(p);
}
void launch_tick(const TickParams& p, bool trace, int grid, int ctas_per_sm, bool tma_sync, cudaStream_t st) {
  const bool small = p.fanout <= 4;          // the common fan-outs (3, 4) get the 4-wide target array
  if (trace) { if (small) launch_tick_v<true, 4>(p, grid, ctas_per_sm, tma_sync, st); else launch_tick_v<true, 8>(p, grid, ctas_per_sm, tma_sync, st); }
  else { if (small) launch_tick_v<false, 4>(p, grid, ctas_per_sm, tma_sync, st); else launch_tick_v<false, 8>(p, grid, ctas_per_sm, tma_sync, st); }
}
// One pass of a tick of an unsharded multi-slot run (SV_PASS): the single-slot kernel on the view the parameter block starts at.
void launch_tick_pass(const TickParams& p, int grid, cudaStream_t st) {
  if (p.fanout <= 4) SFS_LAUNCH(grid, BLOCK, 0, st, tick_kernel<false, 4, false, true, SFS_MB_R1, true>)(p);
  else SFS_LAUNCH(grid, BLOCK, 0, st, tick_kernel<false, 8, false, true, SFS_MB_R1, true>)(p);
}
// The single-view kernel of a dual launch of a sharded run (SV_SINGLE): the single-slot kernel on the one view that has business (multi-slot plane layout).
void launch_tick_single_view(const TickParams& p, int grid, cudaStream_t st) {
  if (p.fanout <= 4) SFS_LAUNCH(grid, BLOCK, 0, st, tick_kernel<false, 4, true, true, SFS_MB_R1S>)(p);
  else SFS_LAUNCH(grid, BLOCK, 0, st, tick_kernel<false, 8, true, true, SFS_MB_R1S>)(p);
}
void launch_fill_idle_rows(u64* rows, u64* grow_rows, u32 n, const u32* sched, bool trace, cudaStream_t st) {
  if (n) SFS_LAUNCH((n + 127) / 128, 128, 0, st, fill_idle_rows_kernel)(rows, grow_rows, n, sched, trace ? 1 : 0);
}
void launch_pushpull(const TickParams& p, const uint4* snap_rec, const u64* snap_node, bool trace, cudaStream_t st) {
  if (trace) SFS_LAUNCH(SFS_SMS * 8, BLOCK, 0, st, pushpull_kernel<true>)(p, snap_rec, snap_node);
  else SFS_LAUNCH(SFS_SMS * 8, BLOCK, 0, st, pushpull_kernel<false>)(p, snap_rec, snap_node);
}
void launch_compute_watch(const u32* row_ptr, const u32* col, const u32* subj_dev, u32 R, u32 first, u32 n_local, u16* watch, cudaStream_t st) {
  SFS_LAUNCH((n_local + 255) / 256, 256, 0, st, compute_watch_kernel)(row_ptr, col, subj_dev, R, first, n_local, watch);
}
void launch_apply_watch(const u16* watch, u32 n_local, u8* busy, u8* hot_static, cudaStream_t st) {
  SFS_LAUNCH((n_local + 255) / 256, 256, 0, st, apply_watch_kernel)(watch, n_local, busy, hot_static);
}
void launch_drain(const DrainParams& p, cudaStream_t st) {
  SFS_LAUNCH(SFS_SMS * 8, BLOCK, 0, st, drain_kernel)(p);
  if (p.byz_on) SFS_LAUNCH(SFS_SMS * 2, BLOCK, 0, st, clear_windows_kernel)(p);
}
void launch_publish(const PublishParams& p, cudaStream_t st) { SFS_LAUNCH(1, 32, 0, st, publish_kernel)(p); }
void launch_init_state(uint4* rec, u64* node_state, u32 n_local, u32 stride, u32 R, u32 init_st, u32 init_clock, cudaStream_t st) {
  SFS_LAUNCH((n_local + 255) / 256, 256, 0, st, init_state_kernel)(rec, node_state, n_local, stride, R, init_st, init_clock);
}
void launch_mark_events(u8* busy, u8* hot_rd, const u32* ev_node, u32 ev_begin, u32 ev_end, u32 first, u32 n_local, cudaStream_t st) {
  const u32 n = ev_end - ev_begin;
  if (!n) return;
  SFS_LAUNCH((n + 127) / 128, 128, 0, st, mark_events_kernel)(busy, hot_rd, ev_node, ev_begin, ev_end, first, n_local);
}
void launch_extract(const uint4* rec, const u64* node_state, u32 n_local, u32 stride, u32 slot, int what, void* out, cudaStream_t st) {
  SFS_LAUNCH((n_local + 255) / 256, 256, 0, st, extract_kernel)(rec, node_state, n_local, stride, slot, what, out);
}
void launch_compose_records(const uint4* rec, const u32* qword, u32 n_local, u32 stride, u32 slot, uint4* out, cudaStream_t st) {
  SFS_LAUNCH((n_local + 255) / 256, 256, 0, st, compose_records_kernel)(rec, qword, n_local, stride, slot, out);
}
void launch_state_hash(const uint4* rec, const u32* qword, const u64* node_state, u32 n_local, u32 stride, u32 first, u32 n_global, u32 R, u64* out, cudaStream_t st) {
  SFS_LAUNCH(SFS_SMS * 4, BLOCK, 0, st, state_hash_kernel)(rec, qword, node_state, n_local, stride, first, n_global, R, out);
}
void launch_summary(const uint4* rec, const u32* qword, const u64* node_state, u32 n_local, u32 stride, u32 first, u32 R, const u32* subj_dev, u64* out, cudaStream_t st) {
  SFS_LAUNCH(SFS_SMS * 4, BLOCK, 0, st, summary_kernel)(rec, qword, node_state, n_local, stride, first, R, subj_dev, out);
}

}  // namespace sfs
