// tests/emu/emu_engine.cpp — fiber scheduler of the CUDA-on-CPU shim (see cuda_runtime.h).  Test infrastructure only.
#include <sched.h>
#include <sys/mman.h>
#include <ctime>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <utility>
#include <vector>

#define SERFSIM_EMU 1
#include "cuda_runtime.h"

#if !defined(__x86_64__)
#error "tests/emu: the fiber switch below is written for x86-64 (System V ABI)"
#endif
// Minimal fiber switch (no signal-mask system call, unlike swapcontext): save the callee-saved registers and the stack
// pointer of the running fiber, load those of the next one.  A new fiber's stack is primed so that the first switch
// "returns" into its entry function.
extern "C" void emu_switch(void** save_sp, void* load_sp);
asm(R"(
.text
.globl emu_switch
.type emu_switch,@function
emu_switch:
  pushq %rbp
  pushq %rbx
  pushq %r12
  pushq %r13
  pushq %r14
  pushq %r15
  movq %rsp, (%rdi)
  movq %rsi, %rsp
  popq %r15
  popq %r14
  popq %r13
  popq %r12
  popq %rbx
  popq %rbp
  ret
.size emu_switch,.-emu_switch
)");

namespace emu {

thread_local LaneCtx* cur = nullptr;
unsigned long probes[32] = {0};
std::atomic<long> live_allocs{0}, fail_countdown{0};

namespace {
constexpr int MAX_THREADS = 1024;
constexpr size_t STACK = 256 * 1024;
struct Lane {
  void* sp = nullptr;        // saved stack pointer while the fiber is not running
  LaneCtx lc;
  bool done = false;
  int wait = 0;              // 0 runnable, 1 warp rendezvous, 2 CTA barrier
  unsigned wait_gen = 0;
  char* stack = nullptr;
};
struct Warp {
  int live = 0, arrived = 0;
  unsigned gen = 0;
  unsigned long long buf[2][32];
  unsigned votes[2];
};
struct Engine {                     // everything a rank thread needs to run kernels; created on first use
  Lane lanes[MAX_THREADS];
  Warp warps[MAX_THREADS / 32];
};
thread_local Engine* eng = nullptr;
#define lanes (eng->lanes)
#define warps (eng->warps)
thread_local int cta_live = 0, cta_arrived = 0;
thread_local unsigned cta_gen = 0;
thread_local void* sched_sp = nullptr;
thread_local Lane* cur_lane = nullptr;
thread_local const std::function<void()>* body = nullptr;

void release_check(Warp& w) { if (w.live > 0 && w.arrived >= w.live) { w.arrived = 0; w.gen++; } }
void cta_release_check() { if (cta_live > 0 && cta_arrived >= cta_live) { cta_arrived = 0; cta_gen++; } }

void lane_entry() {
  (*body)();
  Lane* l = cur_lane;
  l->done = true;
  Warp& w = warps[l->lc.tid.x / 32];
  w.live--; cta_live--;                       // an exited thread no longer takes part in collectives
  release_check(w); cta_release_check();
  emu_switch(&l->sp, sched_sp);
  __builtin_unreachable();                    // a finished fiber is never resumed
}

void warp_rendezvous(Warp& w) {
  Lane* l = cur_lane;
  const unsigned g = w.gen;
  if (++w.arrived >= w.live) { w.arrived = 0; w.gen++; return; }
  l->wait = 1; l->wait_gen = g;
  emu_switch(&l->sp, sched_sp);               // resumed by the scheduler once w.gen has moved on
}
}  // namespace

unsigned lane_id() { return cur_lane->lc.tid.x & 31u; }

void polite_wait(unsigned long spins) {
  sched_yield();
  if (spins > 64 && (spins & 0xfff) == 0) {
    static thread_local time_t t0 = 0;
    static thread_local unsigned long base = 0;
    if (spins < base || !t0) { t0 = time(nullptr); }          // a new wait
    base = spins;
    if (time(nullptr) - t0 > 120) { fprintf(stderr, "emu: a rank has been polling a peer's flag for 120 s — the peer is gone; aborting instead of hanging\n"); abort(); }
  }
}

void cta_barrier() {
  Lane* l = cur_lane;
  const unsigned g = cta_gen;
  if (++cta_arrived >= cta_live) { cta_arrived = 0; cta_gen++; return; }
  l->wait = 2; l->wait_gen = g;
  emu_switch(&l->sp, sched_sp);
}

// Double-buffered by rendezvous generation: a lane can be at most one collective ahead of the slowest lane of its warp.
unsigned long long warp_exchange(unsigned long long v, int x, int abs_lane) {
  Warp& w = warps[cur_lane->lc.tid.x / 32];
  const unsigned lane = lane_id(), par = w.gen & 1u;
  w.buf[par][lane] = v;
  warp_rendezvous(w);
  return w.buf[par][abs_lane >= 0 ? (unsigned)abs_lane : (lane ^ (unsigned)x) & 31u];
}

unsigned warp_ballot(bool pred) {
  Warp& w = warps[cur_lane->lc.tid.x / 32];
  const unsigned lane = lane_id(), par = w.gen & 1u;
  if (w.arrived == 0) w.votes[par] = 0;       // first lane of this collective
  if (pred) w.votes[par] |= 1u << lane;
  warp_rendezvous(w);
  return w.votes[par];
}

unsigned warp_reduce_or(unsigned v) {
  Warp& w = warps[cur_lane->lc.tid.x / 32];
  const unsigned par = w.gen & 1u;
  if (w.arrived == 0) w.votes[par] = 0;
  w.votes[par] |= v;
  warp_rendezvous(w);
  return w.votes[par];
}

void run_grid(unsigned grid, unsigned block, const std::function<void()>& fn) {
  if (block == 0 || block > (unsigned)MAX_THREADS) { fprintf(stderr, "emu: bad block size %u\n", block); abort(); }
  if (cur_lane) { fprintf(stderr, "emu: nested kernel launch\n"); abort(); }
  if (!eng) eng = new Engine();
  body = &fn;
  for (unsigned t = 0; t < block; ++t)
    if (!lanes[t].stack) {
      void* s = mmap(nullptr, STACK, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
      if (s == MAP_FAILED) { perror("emu: mmap"); abort(); }
      lanes[t].stack = (char*)s;
    }
  // CTA order follows SERFSIM_EMU_SCHED too (ascending / reverse / a fresh random permutation per launch): a kernel
  // whose result depends on which CTA runs first is as wrong as one that depends on the lane order.
  static const char* sched_env = getenv("SERFSIM_EMU_SCHED");
  static thread_local std::vector<unsigned> cta_order;
  static thread_local unsigned long long cta_rng = 0x243F6A8885A308D3ull;
  cta_order.resize(grid);
  for (unsigned b = 0; b < grid; ++b) cta_order[b] = (sched_env && !strcmp(sched_env, "reverse")) ? grid - 1 - b : b;
  if (sched_env && !strncmp(sched_env, "random", 6))
    for (unsigned b = grid; b > 1; --b) {
      cta_rng ^= cta_rng >> 12; cta_rng ^= cta_rng << 25; cta_rng ^= cta_rng >> 27;
      std::swap(cta_order[b - 1], cta_order[(unsigned)(((cta_rng * 0x2545F4914F6CDD1Dull) >> 33) % b)]);
    }
  for (unsigned bi = 0; bi < grid; ++bi) {
    const unsigned b = cta_order[bi];
    const unsigned nw = (block + 31) / 32;
    for (unsigned w = 0; w < nw; ++w) { warps[w].live = 0; warps[w].arrived = 0; warps[w].gen = 0; }
    cta_live = (int)block; cta_arrived = 0; cta_gen = 0;
    for (unsigned t = 0; t < block; ++t) {
      Lane& l = lanes[t];
      l.done = false; l.wait = 0;
      l.lc.tid = uint3{t, 0, 0}; l.lc.bid = uint3{b, 0, 0}; l.lc.bdim = uint3{block, 1, 1}; l.lc.gdim = uint3{grid, 1, 1};
      warps[t / 32].live++;
      // prime the stack: six callee-saved registers (zero), then lane_entry as the address emu_switch returns to; the
      // slot above it is the (never used) return address of lane_entry, which puts rsp at 16n + 8 on entry as the ABI asks
      void** top = reinterpret_cast<void**>(l.stack + STACK);
      top[-1] = nullptr;
      top[-2] = reinterpret_cast<void*>(&lane_entry);
      for (int k = 3; k <= 8; ++k) top[-k] = nullptr;
      l.sp = &top[-8];
    }
    unsigned remaining = block;
    // Lane order of a scheduling pass.  Default: ascending thread index.  SERFSIM_EMU_SCHED=reverse | random:<seed>
    // visits the lanes in another order (re-drawn every pass for `random`): results must not depend on it, so running
    // the parity suites under several schedules is a cheap check for order-dependent (racy) kernel logic.
    static thread_local std::vector<unsigned> order;
    order.resize(block);
    for (unsigned t = 0; t < block; ++t) order[t] = t;
    static const char* sched = getenv("SERFSIM_EMU_SCHED");
    static thread_local unsigned long long rng = 0;
    const bool random = sched && !strncmp(sched, "random", 6);
    if (random && !rng) rng = 0x9E3779B97F4A7C15ull ^ (strlen(sched) > 7 ? strtoull(sched + 7, nullptr, 10) * 0xD1B54A32D192ED03ull : 1);
    if (sched && !strcmp(sched, "reverse")) for (unsigned t = 0; t < block; ++t) order[t] = block - 1 - t;
    while (remaining) {
      bool progressed = false;
      if (random)
        for (unsigned t = block - 1; t > 0; --t) {          // Fisher–Yates with xorshift64*
          rng ^= rng >> 12; rng ^= rng << 25; rng ^= rng >> 27;
          const unsigned j = (unsigned)(((rng * 0x2545F4914F6CDD1Dull) >> 33) % (t + 1));
          std::swap(order[t], order[j]);
        }
      for (unsigned k = 0; k < block; ++k) {
        const unsigned t = order[k];
        Lane& l = lanes[t];
        if (l.done) continue;
        if (l.wait == 1 && warps[t / 32].gen == l.wait_gen) continue;
        if (l.wait == 2 && cta_gen == l.wait_gen) continue;
        l.wait = 0;
        cur_lane = &l; cur = &l.lc;
        emu_switch(&sched_sp, l.sp);
        progressed = true;
        if (l.done) --remaining;
      }
      if (!progressed) { fprintf(stderr, "emu: deadlock — a collective is waiting for threads that never arrive (block %u)\n", b); abort(); }
    }
  }
  cur_lane = nullptr; cur = nullptr; body = nullptr;
}

}  // namespace emu

extern "C" __attribute__((visibility("default"))) unsigned long emu_probe(int i) { return emu::probes[i & 31]; }
extern "C" __attribute__((visibility("default"))) void emu_probe_reset() { for (auto& p : emu::probes) p = 0; }
// Resources alive now (cuda_runtime.h: live_allocs), and k >= 1: the k-th next allocation, stream or event creation fails with
// cudaErrorMemoryAllocation (0: none).
extern "C" __attribute__((visibility("default"))) long emu_live_allocs() { return emu::live_allocs.load(); }
extern "C" __attribute__((visibility("default"))) void emu_fail_alloc_at(long k) { emu::fail_countdown.store(k); }
