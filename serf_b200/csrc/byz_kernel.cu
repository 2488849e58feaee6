// byz_kernel.cu — byzantine stale-record injectors (BASELINE configs[4]); model and rules in byz.cuh.
//
// One launch per tick AFTER the membership tick kernel: one thread per byzantine node reads its end-of-tick views
// (32 B per subject), re-draws this tick's gossip peers (same Philox block as the tick kernel), RED.MAXes the stale
// entries into the inbox planes the tick kernel just filled (value + 1 encoding, same planes, same reduction), marks the
// destination tile hot, and judges the entry against the receiver's end-of-tick record (one 32-byte gather per
// (peer, subject)) to raise its OWN anomaly flag — a thread writes only its own flag, no atomics on that path.
// At 1 % injectors and fan-out 4 this is ≈ 4 % of a plateau tick's gathers.
#include "tick_kernel.cuh"   // first: brings in <cuda_runtime.h> (nvcc's own, or the host shim of tests/emu)
#include "byz.cuh"
#include "uevent.cuh"

namespace sfs {
namespace {

__global__ void __launch_bounds__(128) byz_kernel(const __grid_constant__ ByzParams p) {
  if (p.gate && *p.gate) return;                               // the run is over (convergence gate): this tick does not exist
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  u32 n_msgs = 0, n_edges = 0, kL = 0, kJ = 0, kM = 0;
  bool wrote_remote = false;
  if (i < p.n_byz) {
    const u32 u = p.ids[i];
    const u32 ul = u - p.first;
    const u64 ns = p.node_state[ul];
    if (nw_up(ns)) {                                           // up after this tick's operations
      const u32 row0 = p.row_ptr[ul], deg = p.row_ptr[ul + 1] - row0;
      u32 tg[MAX_FANOUT];
      const u32 nt = ue_pick_targets(p.tick, u, row0, deg, p.fanout, p.seed_lo, p.seed_hi, p.col, tg);
      bool flag = false;
      for (u32 s = 0; s < p.R; ++s) {
        Rec r;
        unpack(load_rec(p.rec, (size_t)s * p.stride + ul), r);
        const ByzEntries e = byz_entries(r, p.delta);
        if (!e.any) continue;
        u32* const planeS = p.inbox_wr + (size_t)(e.serf_kind * p.R + s) * p.stride;
        const u32 serf_val1 = (e.serf_kind == KIND_LEAVE ? leave_key(e.serf_lt, false) : e.serf_lt) + 1u;   // the word an honest sender would post
        u32* const planeM = p.inbox_wr + (size_t)(KIND_ML * p.R + s) * p.stride;
        for (u32 k = 0; k < nt; ++k) {
          const u32 dl = tg[k] - p.first;
          n_msgs += 2; n_edges += 1;
          if (p.snd.world > 1 && dl >= p.n_local) {                // the peer lives in another shard: triple into its window
            const ShardIdx t = shard_of(tg[k], p.snd.shard_size, p.snd.shard_inv);
            const u32 dloc = t.local | BYZ_FLAG;
            win_append<3>(p.snd, p.overflow, t.shard, {win_entry(serf_val1, s, e.serf_kind, dloc), win_entry(e.ml_key + 1u, s, KIND_ML, dloc),
                                     win_entry(u + 1u, BYZ_ANNOT_SLOT, KIND_EXTRA, dloc)});
            wrote_remote = true;
            continue;                                          // kinds / tile flags / verdict are the receiving shard's business
          }
          atomicMax(planeS + dl, serf_val1);
          atomicMax(planeM + dl, e.ml_key + 1u);
          p.hot_wr[dl >> TILE_SHIFT] = 1;                      // the destination tile must run next tick
          if (e.serf_kind == KIND_LEAVE) ++kL; else ++kJ;
          ++kM;
          if (nw_up(p.node_state[dl])) {                       // the receiver is up when the packet arrives
            Rec q;
            unpack(load_rec(p.rec, (size_t)s * p.stride + dl), q);
            flag |= byz_anomalous(q, e, p.delta);
          }
        }
      }
      if (flag) p.anomaly[ul] = 1;
    }
  }
  if (wrote_remote) __threadfence_system();   // peer-window stores are performed before the publish kernel raises the flags
  // warp sums → a few atomics per warp
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    n_msgs += __shfl_xor_sync(0xffffffffu, n_msgs, o); n_edges += __shfl_xor_sync(0xffffffffu, n_edges, o);
    kL += __shfl_xor_sync(0xffffffffu, kL, o); kJ += __shfl_xor_sync(0xffffffffu, kJ, o); kM += __shfl_xor_sync(0xffffffffu, kM, o);
  }
  if ((threadIdx.x & 31) == 0) {
    typedef unsigned long long ull;
    if (n_msgs) atomicAdd((ull*)(p.totals + 0), (ull)n_msgs);
    if (n_edges) atomicAdd((ull*)(p.totals + 1), (ull)n_edges);
    if (kL) atomicAdd(p.kinds_cur + KIND_LEAVE, kL);
    if (kJ) atomicAdd(p.kinds_cur + KIND_JOIN, kJ);
    if (kM) atomicAdd(p.kinds_cur + KIND_ML, kM);
  }
}

}  // namespace

void launch_byz(const ByzParams& p, cudaStream_t st) {
  if (!p.n_byz) return;
  SFS_LAUNCH((p.n_byz + 127) / 128, 128, 0, st, byz_kernel)(p);
}

}  // namespace sfs
