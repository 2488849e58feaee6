// uevent_kernel.cu — user-event dissemination tick (SURVEY §8f row 3); rules and reference citations in uevent.cuh.
//
// One launch per tick, BEFORE the membership tick kernel (it needs the node's pre-operation up flag and the op bit of
// the busy byte, both consumed by that kernel; the two kernels touch disjoint state, so their order is otherwise free).
// One thread per node, grid-stride: 4 B inbox word + 16 B event record in; a node with nothing arrived, nothing
// queued and no host operation stops after those 20 bytes.  Sends are one RED.OR per (target, tick) into the other
// parity's inbox plane.  Counters go to the same trace row the membership kernel fills (edge_updates, messages,
// changed, pending, hash), so the convergence logic sees user events with no extra host code, plus run totals.
#include "tick_kernel.cuh"   // first: brings in <cuda_runtime.h> (nvcc's own, or the host shim of tests/emu)
#include "uevent.cuh"

namespace sfs {
namespace {

constexpr int UE_BLOCK = 256;

__device__ __forceinline__ u32 ue_warp_sum(u32 v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ u64 ue_warp_sum64(u64 v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <bool TRACE>
__global__ void __launch_bounds__(UE_BLOCK) uevent_kernel(const __grid_constant__ UeParams p) {
  if (gate_closed(p.gate, blockIdx.x == 0 && threadIdx.x == 0)) return;   // the run is over: this tick does not exist
  if (tick_is_idle(p.sched, p.tick, p.ev_begin, p.ev_end)) return;          // nothing can happen in this tick (the membership kernel writes its row)
  UeCounts c = {};
  u32 changed = 0;
  u64 hash = 0;
  bool wrote_remote = false;
  for (u32 vl = blockIdx.x * UE_BLOCK + threadIdx.x; vl < p.n_local; vl += gridDim.x * UE_BLOCK) {
    const u32 v = p.first + vl;
    const u32 arrived = p.inbox_rd[vl];
    if (arrived) p.inbox_rd[vl] = 0;                           // consumed; this parity is written again two ticks from now
    const u32 busy = p.busy[vl];
    const uint4 w0 = p.state[vl];
    const bool queued = (w0.z | w0.w) != 0;
    if (!TRACE && !arrived && !(busy & BUSY_OP) && !queued) continue;
    UeRec r;
    ue_unpack(w0, r);
    const u64 ns = p.node_state[vl];
    const bool up_r = nw_up(ns);
    u32 op = 0, op_slot = 0;
    if (busy & BUSY_OP) op = host_op_of(p, v, op_slot);
    bool up_s = up_r;
    if (op == OP_FAIL) up_s = false;
    if (op == OP_REJOIN) up_s = true;

    const u32 delivered0 = c.delivered;
    bool stamped = false;
    const u32 L = ue_receive_and_originate(r, arrived, up_r, op, op_slot, p.ltime, p.table, p.limit, c, stamped);
    if (stamped) p.ltime[op_slot] = L;                         // read by receivers from the next tick on
    changed += c.delivered - delivered0;

    if (up_s && ue_queued(r, p.table.n)) {
      const u32 row0 = p.row_ptr[vl], deg = p.row_ptr[vl + 1] - row0;
      u32 tg[MAX_FANOUT];
      const u32 nt = ue_pick_targets(p.tick, v, row0, deg, p.fanout, p.seed_lo, p.seed_hi, p.col, tg);
      u32 bits[MAX_FANOUT];
      c.messages += ue_plan_send<(int)MAX_FANOUT>(r, p.table.n, nt, bits);
      for (u32 k = 0; k < nt; ++k) {
        if (!bits[k]) continue;
        c.edges++;
        const u32 dl = tg[k] - p.first;
        if (p.snd.world == 1 || dl < p.n_local) { atomicOr(p.inbox_wr + dl, bits[k]); continue; }
        // another shard owns the target: one 8-byte entry per event into its window (slot = event, value = ltime + 1)
        const ShardIdx t = shard_of(tg[k], p.snd.shard_size, p.snd.shard_inv);
        for (u32 e = 0; e < p.table.n; ++e) {
          if (!((bits[k] >> e) & 1u)) continue;
          const u32 Le = (stamped && e == op_slot) ? L : p.ltime[e];
          win_append<1>(p.snd, p.overflow, t.shard, {win_entry(Le + 1u, e, KIND_EXTRA, t.local)});
          wrote_remote = true;
        }
      }
    }
    if (up_s) c.pending += ue_queued(r, p.table.n);           // a crashed node's queue is frozen, not pending
    const uint4 w1 = ue_pack(r);
    if ((w1.x ^ w0.x) | (w1.y ^ w0.y) | (w1.z ^ w0.z) | (w1.w ^ w0.w)) p.state[vl] = w1;
    if (TRACE) hash += ue_hash((u64)(p.R + 1) * p.n_global + v, w1);
    if (r.clock >= LTIME_LIMIT) *p.overflow = 1;
  }
  if (wrote_remote) __threadfence_system();   // peer-window stores are performed before the publish kernel raises the flags
  // warp sums, one atomic per warp and counter (this kernel is not the hot path; the row is shared with the tick kernel)
  const u32 lane = threadIdx.x & 31;
  const u32 s_msgs = ue_warp_sum(c.messages), s_edges = ue_warp_sum(c.edges), s_deliv = ue_warp_sum(c.delivered),
            s_dup = ue_warp_sum(c.duplicates), s_old = ue_warp_sum(c.too_old), s_pend = ue_warp_sum(c.pending), s_chg = ue_warp_sum(changed);
  const u64 s_hash = TRACE ? ue_warp_sum64(hash) : 0;
  if (lane == 0) {
    typedef unsigned long long ull;
    if (s_edges) { atomicAdd((ull*)(p.row + ROW_EDGES), (ull)s_edges); atomicAdd((ull*)(p.totals + 1), (ull)s_edges); }
    if (s_msgs) { atomicAdd((ull*)(p.row + ROW_MESSAGES), (ull)s_msgs); atomicAdd((ull*)(p.totals + 0), (ull)s_msgs); }
    if (s_chg) atomicAdd((ull*)(p.row + ROW_CHANGED), (ull)s_chg);
    if (s_pend) atomicAdd((ull*)(p.row + ROW_PENDING), (ull)s_pend);
    if (s_pend | s_msgs) atomicAdd(p.sched + SCHED_UE_ACTIVITY, 1u);      // queued or sent events: the next tick cannot be skipped
    if (s_deliv) atomicAdd((ull*)(p.totals + 2), (ull)s_deliv);
    if (s_dup) atomicAdd((ull*)(p.totals + 3), (ull)s_dup);
    if (s_old) atomicAdd((ull*)(p.totals + 4), (ull)s_old);
    if (TRACE && s_hash) atomicAdd((ull*)(p.row + ROW_HASH), (ull)s_hash);
  }
}

__global__ void ue_init_kernel(uint4* state, u32 n_local) {
  const u32 vl = blockIdx.x * blockDim.x + threadIdx.x;
  if (vl < n_local) state[vl] = make_uint4(UE_INIT_CLOCK, 0u, 0u, 0u);
}

// what: 0 event clock (u64 out), 1 seen flag of event `e` (u8 out)
__global__ void ue_extract_kernel(const uint4* state, u32 n_local, int what, u32 e, void* out) {
  const u32 vl = blockIdx.x * blockDim.x + threadIdx.x;
  if (vl >= n_local) return;
  const uint4 w = state[vl];
  if (what == 0) reinterpret_cast<u64*>(out)[vl] = w.x;
  else reinterpret_cast<u8*>(out)[vl] = (u8)((w.y >> e) & 1u);
}

// out[0] += queued broadcasts, out[1] = max event clock, out[2] += Σ ue_hash
__global__ void __launch_bounds__(UE_BLOCK) ue_summary_kernel(const uint4* state, u32 n_local, u32 first, u32 n_global, u32 R, u32 n_events, u64* out) {
  u32 queued = 0, mx = 0;
  u64 h = 0;
  for (u32 vl = blockIdx.x * UE_BLOCK + threadIdx.x; vl < n_local; vl += gridDim.x * UE_BLOCK) {
    const uint4 w = state[vl];
    UeRec r;
    ue_unpack(w, r);
    queued += ue_queued(r, n_events);
    mx = max(mx, r.clock);
    h += ue_hash((u64)(R + 1) * n_global + first + vl, w);
  }
  queued = ue_warp_sum(queued);
  h = ue_warp_sum64(h);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) {
    typedef unsigned long long ull;
    if (queued) atomicAdd((ull*)(out + 0), (ull)queued);
    atomicMax((ull*)(out + 1), (ull)mx);
    if (h) atomicAdd((ull*)(out + 2), (ull)h);
  }
}

}  // namespace

void launch_uevent(const UeParams& p, bool trace, cudaStream_t st) {
  const int grid = SFS_SMS * 8;
  if (trace) SFS_LAUNCH(grid, UE_BLOCK, 0, st, uevent_kernel<true>)(p);
  else SFS_LAUNCH(grid, UE_BLOCK, 0, st, uevent_kernel<false>)(p);
}
void launch_ue_init(uint4* state, u32 n_local, cudaStream_t st) { SFS_LAUNCH((n_local + 255) / 256, 256, 0, st, ue_init_kernel)(state, n_local); }
void launch_ue_extract(const uint4* state, u32 n_local, int what, u32 e, void* out, cudaStream_t st) {
  SFS_LAUNCH((n_local + 255) / 256, 256, 0, st, ue_extract_kernel)(state, n_local, what, e, out);
}
void launch_ue_summary(const uint4* state, u32 n_local, u32 first, u32 n_global, u32 R, u32 n_events, u64* out, cudaStream_t st) {
  SFS_LAUNCH(SFS_SMS * 4, UE_BLOCK, 0, st, ue_summary_kernel)(state, n_local, first, n_global, R, n_events, out);
}

}  // namespace sfs
