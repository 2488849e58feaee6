// Can a delivered-bitmap in front of the inbox save scattered RED.MAX?  In a saturated tick every sender of a wave sends the
// same value for a (kind, view), and a destination receives about Poisson(fanout) of them: three REDs in four write a value the
// word already holds.  This benchmark compares, for n destinations and 4·n deliveries with uniform random targets, all of one value:
//   plain      RED.MAX evict_last into a 4·n-byte plane (what the tick kernel does);
//   filter/ld  a scattered load of the destination's bit in an n/8-byte bitmap; bit clear → RED.OR the bit, RED.MAX the value;
//   filter/atom ATOM.OR with return on the bit; it was clear → RED.MAX the value;
//   filter/ld weak  as filter/ld with a weak load, which L1 may serve (a stale clear bit only costs a duplicate RED);
// alone, and next to a grid-stride copy kernel on a second stream that moves about 1.7 GB (read + write), a stand-in for the
// streamed planes of a saturated pass.  Both kernels are sized to be co-resident (4 + 2 CTAs of 256 threads per SM).  The
// results are in DESIGN §5 ("Sends skip the REDs that cannot raise the word"), next to the filter the tick kernel took instead.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/ubench/red_dedup tools/ubench/red_dedup.cu
//   tools/ubench/red_dedup [n]           (on the GPU)
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

typedef uint32_t u32;
typedef uint64_t u64;

__device__ __forceinline__ u32 mix(u32 x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }
__device__ __forceinline__ u64 pol_last() { u64 p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ u64 pol_first() { u64 p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }

enum { PLAIN = 0, FILT_LD = 1, FILT_ATOM = 2, FILT_LD_WEAK = 3 };
constexpr int PER_NODE = 4;
constexpr u32 VAL = 0x1234u;

// Grid-stride over the senders (grid = 132 · 4 CTAs: the same co-residency the concurrent case needs).  count != null: a
// separate, untimed run that counts the REDs into the plane that were issued.
template <int MODE>
__global__ void __launch_bounds__(256) scatter(u32 n, u32* plane, u32* bits, u32 salt, unsigned long long* count) {
  const u64 pl = pol_last();
  u32 issued = 0;
  for (u32 v = blockIdx.x * 256 + threadIdx.x; v < n; v += gridDim.x * 256) {
    const u32 h = mix(v ^ salt);
#pragma unroll
    for (int j = 0; j < PER_NODE; ++j) {
      const u32 tg = __umulhi(mix(h + j), n);
      u32* ptr = plane + tg;
      u32* bw = bits + (tg >> 5);
      const u32 bit = 1u << (tg & 31);
      bool go = true;
      if (MODE == FILT_LD || MODE == FILT_LD_WEAK) {
        u32 w;
        if (MODE == FILT_LD) asm volatile("ld.relaxed.gpu.global.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(w) : "l"(bw), "l"(pl) : "memory");
        else asm volatile("ld.global.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(w) : "l"(bw), "l"(pl) : "memory");
        go = !(w & bit);
        if (go) asm volatile("red.relaxed.gpu.global.or.L2::cache_hint.b32 [%0], %1, %2;" :: "l"(bw), "r"(bit), "l"(pl) : "memory");
      } else if (MODE == FILT_ATOM) {
        u32 old;
        asm volatile("atom.relaxed.gpu.global.or.L2::cache_hint.b32 %0, [%1], %2, %3;" : "=r"(old) : "l"(bw), "r"(bit), "l"(pl) : "memory");
        go = !(old & bit);
      }
      if (go) { asm volatile("red.relaxed.gpu.global.max.L2::cache_hint.u32 [%0], %1, %2;" :: "l"(ptr), "r"(VAL), "l"(pl) : "memory"); ++issued; }
    }
  }
  if (count) atomicAdd(count, (unsigned long long)issued);
}

// Streamed planes of a pass: read n16 16-byte words with evict_first, write them elsewhere.
__global__ void __launch_bounds__(256) stream_copy(const uint4* src, uint4* dst, size_t n16) {
  const u64 pf = pol_first();
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n16; i += (size_t)gridDim.x * 256) {
    uint4 x;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;" : "=r"(x.x), "=r"(x.y), "=r"(x.z), "=r"(x.w) : "l"(src + i), "l"(pf));
    asm volatile("st.global.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;" :: "l"(dst + i), "r"(x.x), "r"(x.y), "r"(x.z), "r"(x.w), "l"(pf) : "memory");
  }
}

static void check(cudaError_t e, const char* what) { if (e != cudaSuccess) { printf("CUDA error %s: %s\n", what, cudaGetErrorString(e)); exit(1); } }

struct Ctx { u32 n; u32 *plane, *bits; uint4 *src, *dst; size_t n16; cudaStream_t s0, s1; cudaEvent_t a, b, j; unsigned long long* count; };

static void launch_scatter(Ctx& c, int mode, u32 salt, unsigned long long* count) {
  const int grid = 132 * 4;
  if (mode == PLAIN) scatter<PLAIN><<<grid, 256, 0, c.s0>>>(c.n, c.plane, c.bits, salt, count);
  else if (mode == FILT_LD) scatter<FILT_LD><<<grid, 256, 0, c.s0>>>(c.n, c.plane, c.bits, salt, count);
  else if (mode == FILT_ATOM) scatter<FILT_ATOM><<<grid, 256, 0, c.s0>>>(c.n, c.plane, c.bits, salt, count);
  else scatter<FILT_LD_WEAK><<<grid, 256, 0, c.s0>>>(c.n, c.plane, c.bits, salt, count);
}

// mode < 0: the copy kernel alone; with_stream: the copy kernel runs concurrently on s1.  Returns the mean over reps (ms) and the best.
static void timed(Ctx& c, int mode, bool with_stream, double& mean, double& best) {
  const int reps = 10;
  mean = 0; best = 1e30;
  for (int r = 0; r < reps + 2; ++r) {
    check(cudaMemsetAsync(c.plane, 0, (size_t)c.n * 4, c.s0), "memset plane");       // a fresh launch: nothing delivered yet
    check(cudaMemsetAsync(c.bits, 0, (size_t)(c.n + 31) / 32 * 4, c.s0), "memset bits");
    check(cudaEventRecord(c.a, c.s0), "record");
    check(cudaStreamWaitEvent(c.s1, c.a, 0), "wait");
    if (with_stream || mode < 0) stream_copy<<<132 * 2, 256, 0, c.s1>>>(c.src, c.dst, c.n16);
    if (mode >= 0) launch_scatter(c, mode, 77 + r, nullptr);
    check(cudaEventRecord(c.j, c.s1), "record");
    check(cudaStreamWaitEvent(c.s0, c.j, 0), "wait");
    check(cudaEventRecord(c.b, c.s0), "record");
    check(cudaEventSynchronize(c.b), "sync");
    float ms = 0;
    cudaEventElapsedTime(&ms, c.a, c.b);
    if (r >= 2) { mean += ms / reps; if (ms < best) best = ms; }
  }
  check(cudaGetLastError(), "launch");
}

int main(int argc, char** argv) {
  Ctx c;
  c.n = argc > 1 ? (u32)atoll(argv[1]) : 10000000u;
  const size_t stream_bytes = 850ull << 20;          // read 850 MB + write 850 MB ≈ 1.7 GB moved
  c.n16 = stream_bytes / 16;
  check(cudaMalloc(&c.plane, (size_t)c.n * 4), "malloc");
  check(cudaMalloc(&c.bits, (size_t)(c.n + 31) / 32 * 4), "malloc");
  check(cudaMalloc(&c.src, stream_bytes), "malloc");
  check(cudaMalloc(&c.dst, stream_bytes), "malloc");
  check(cudaMalloc(&c.count, 8), "malloc");
  check(cudaMemset(c.src, 1, stream_bytes), "memset");
  cudaStreamCreateWithFlags(&c.s0, cudaStreamNonBlocking);
  cudaStreamCreateWithFlags(&c.s1, cudaStreamNonBlocking);
  cudaEventCreate(&c.a); cudaEventCreate(&c.b); cudaEventCreate(&c.j);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  printf("# %s, %u destinations, %u deliveries (uniform random, one value), plane %.1f MB, bitmap %.2f MB\n", prop.name, c.n,
         c.n * PER_NODE, c.n * 4 / 1e6, c.n / 8 / 1e6);
  const char* names[4] = {"plain RED.MAX evict_last", "filter: LDG bit, RED.OR + RED.MAX", "filter: ATOM.OR bit, RED.MAX", "filter: weak LDG bit, RED.OR + RED.MAX"};
  double m, b, sm, sb;
  timed(c, -1, true, sm, sb);
  printf("%-40s %9.1f us (best %8.1f)  %.2f TB/s\n", "copy kernel alone (1.78 GB moved)", 1e3 * sm, 1e3 * sb, 2.0 * stream_bytes / (sm * 1e-3) / 1e12);
  double plain_alone = 0, plain_conc = 0;
  // plain runs first and last: the spread between its two runs is the noise the others are read against
  const int order[5] = {PLAIN, FILT_LD, FILT_ATOM, FILT_LD_WEAK, PLAIN};
  for (int mode : order) {
    check(cudaMemsetAsync(c.plane, 0, (size_t)c.n * 4, c.s0), "memset");
    check(cudaMemsetAsync(c.bits, 0, (size_t)(c.n + 31) / 32 * 4, c.s0), "memset");
    check(cudaMemsetAsync(c.count, 0, 8, c.s0), "memset");
    launch_scatter(c, mode, 76, c.count);
    check(cudaStreamSynchronize(c.s0), "sync");
    unsigned long long issued = 0;
    check(cudaMemcpy(&issued, c.count, 8, cudaMemcpyDeviceToHost), "copy");
    timed(c, mode, false, m, b);
    if (mode == PLAIN && plain_alone == 0) plain_alone = m;
    printf("%-40s %9.1f us (best %8.1f)  alone      %5.1f %% of plain   RED.MAX issued %.1f %%\n", names[mode], 1e3 * m, 1e3 * b,
           100.0 * m / plain_alone, 100.0 * issued / ((double)c.n * PER_NODE));
    timed(c, mode, true, m, b);
    const double added = m - sm;
    if (mode == PLAIN && plain_conc == 0) plain_conc = added;
    printf("%-40s %9.1f us (best %8.1f)  with copy: +%7.1f us over the copy alone, %5.1f %% of plain\n", names[mode], 1e3 * m, 1e3 * b, 1e3 * added,
           100.0 * added / plain_conc);
  }
  return 0;
}
