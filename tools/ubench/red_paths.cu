// Where does the scattered-RED floor of the tick kernel come from?  (4 scattered RED.MAX per node are the largest share of
// a plateau tick.)  This benchmark separates
//   * SM side (LSU / L1tex wavefronts) from L2 side (atomic units): the same work on 132, 66 and 33 SMs — an SM-side limit
//     scales with the number of SMs, an L2-side limit does not;
//   * the operation: RED.MAX vs RED.ADD vs plain scattered STG.32 vs scattered LDG.32, with / without the evict_last hint;
//   * the footprint: a 4 MB / 40 MB plane (L2 resident) vs 240 MB (the two-slot bench workload's six planes);
//   * occupancy: 1, 2, 4, 8 CTAs of 256 threads per SM;
//   * locality: targets confined to a 1 MB window that moves with the node id (what a small-world graph's ring
//     neighbours look like) vs uniformly random targets.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/ubench/red_paths tools/ubench/red_paths.cu
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

typedef uint32_t u32;
typedef uint64_t u64;

__device__ __forceinline__ u32 mix(u32 x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }
__device__ __forceinline__ u64 pol_last() { u64 p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ u32 smid() { u32 r; asm volatile("mov.u32 %0, %%smid;" : "=r"(r)); return r; }

enum { OP_RED_MAX_HINT = 0, OP_RED_MAX = 1, OP_RED_ADD = 2, OP_STG = 3, OP_LDG = 4 };

// CTAs that land on an SM >= sm_limit leave at once; the others share the node range through an atomic work counter
// (chunks of 256 nodes), so the SAME total work runs on fewer SMs.  window = 0: targets uniform over [0, span);
// window > 0: targets uniform over [v - window/2, v + window/2) (mod span).
template <int OP, int PER_NODE>
__global__ void __launch_bounds__(256) k(u32 n, u32 span, u32 window, u32* plane, u32 salt, u32 sm_limit, u32* work, u32* sink) {
  if (smid() >= sm_limit) return;
  const u64 pl = pol_last();
  __shared__ u32 chunk_s;
  u32 acc = 0;
  for (;;) {
    __syncthreads();
    if (threadIdx.x == 0) chunk_s = atomicAdd(work, 1u);
    __syncthreads();
    const u32 chunk = chunk_s;
    if ((u64)chunk * 256 >= n) break;
    const u32 v = chunk * 256 + threadIdx.x;
    if (v >= n) continue;
    const u32 h = mix(v ^ salt);
#pragma unroll
    for (int j = 0; j < PER_NODE; ++j) {
      const u32 r = mix(h + j);
      u32 tg;
      if (window) { tg = (u32)(((u64)v * span) / n) + __umulhi(r, window) + span - (window >> 1); tg %= span; }
      else tg = __umulhi(r, span);
      u32* ptr = plane + tg;
      if (OP == OP_RED_MAX_HINT) asm volatile("red.relaxed.gpu.global.max.L2::cache_hint.u32 [%0], %1, %2;" :: "l"(ptr), "r"(v + 1), "l"(pl) : "memory");
      else if (OP == OP_RED_MAX) asm volatile("red.relaxed.gpu.global.max.u32 [%0], %1;" :: "l"(ptr), "r"(v + 1) : "memory");
      else if (OP == OP_RED_ADD) asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" :: "l"(ptr), "r"(1u) : "memory");
      else if (OP == OP_STG) asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" :: "l"(ptr), "r"(v + 1) : "memory");
      else { u32 x; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(x) : "l"(ptr)); acc += x; }
    }
  }
  if (acc == 0xdeadbeefu) *sink = acc;
}

static double g_clk_ghz = 1.965;

template <int OP, int PER_NODE>
static void run(const char* name, u32 n, u32 span, u32 window, u32* plane, u32* work, u32* sink, int ctas_per_sm, u32 sm_limit) {
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  const int grid = 132 * ctas_per_sm;
  const int reps = 6;
  float best = 1e30f, tot = 0;
  for (int r = 0; r < reps + 2; ++r) {
    cudaMemsetAsync(work, 0, 4);
    cudaEventRecord(a);
    k<OP, PER_NODE><<<grid, 256>>>(n, span, window, plane, 100 + r, sm_limit, work, sink);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    if (r >= 2) { tot += ms; if (ms < best) best = ms; }
  }
  const double us = 1e3 * tot / reps;
  const double ops = (double)n * PER_NODE;
  printf("%-58s sms %3u  ctas/sm %d  %8.1f us (best %7.1f)  %6.1f Gop/s  %5.2f SM-cycles/lane\n", name, sm_limit, ctas_per_sm, us, 1e3 * best,
         ops / us * 1e-3, us * 1e-6 * g_clk_ghz * 1e9 * sm_limit / ops);
  if (cudaGetLastError() != cudaSuccess) { printf("CUDA error\n"); exit(1); }
}

int main(int argc, char** argv) {
  const u32 n = argc > 1 ? (u32)atoll(argv[1]) : 10000000u;
  const u32 big = 60000000u;                        // 240 MB of u32
  u32 *plane, *work, *sink;
  cudaMalloc(&plane, (size_t)big * 4); cudaMalloc(&work, 4); cudaMalloc(&sink, 4);
  cudaMemset(plane, 0, (size_t)big * 4);
  int clk_khz = 0;
  cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
  if (clk_khz > 0) g_clk_ghz = clk_khz * 1e-6;
  printf("# n = %u nodes, 4 scattered ops per node unless stated, 256-thread CTAs, SM clock %.3f GHz (nominal max)\n", n, g_clk_ghz);
  printf("## operation (40 MB plane, 132 SMs, 4 CTAs/SM)\n");
  run<OP_RED_MAX_HINT, 4>("RED.MAX evict_last", n, n, 0, plane, work, sink, 4, 132);
  run<OP_RED_MAX, 4>("RED.MAX", n, n, 0, plane, work, sink, 4, 132);
  run<OP_RED_ADD, 4>("RED.ADD", n, n, 0, plane, work, sink, 4, 132);
  run<OP_STG, 4>("STG.32", n, n, 0, plane, work, sink, 4, 132);
  run<OP_LDG, 4>("LDG.32", n, n, 0, plane, work, sink, 4, 132);
  printf("## SM count (RED.MAX evict_last, 40 MB plane, 4 CTAs/SM): SM-side limit scales, L2-side limit does not\n");
  run<OP_RED_MAX_HINT, 4>("RED.MAX evict_last", n, n, 0, plane, work, sink, 4, 99);
  run<OP_RED_MAX_HINT, 4>("RED.MAX evict_last", n, n, 0, plane, work, sink, 4, 66);
  run<OP_RED_MAX_HINT, 4>("RED.MAX evict_last", n, n, 0, plane, work, sink, 4, 33);
  run<OP_STG, 4>("STG.32", n, n, 0, plane, work, sink, 4, 66);
  run<OP_LDG, 4>("LDG.32", n, n, 0, plane, work, sink, 4, 66);
  printf("## occupancy (RED.MAX evict_last, 40 MB plane, 132 SMs)\n");
  run<OP_RED_MAX_HINT, 4>("RED.MAX evict_last", n, n, 0, plane, work, sink, 1, 132);
  run<OP_RED_MAX_HINT, 4>("RED.MAX evict_last", n, n, 0, plane, work, sink, 2, 132);
  run<OP_RED_MAX_HINT, 4>("RED.MAX evict_last", n, n, 0, plane, work, sink, 8, 132);
  printf("## footprint (RED.MAX evict_last, 132 SMs, 4 CTAs/SM)\n");
  run<OP_RED_MAX_HINT, 4>("4 MB plane", n, 1000000u, 0, plane, work, sink, 4, 132);
  run<OP_RED_MAX_HINT, 4>("80 MB", n, 20000000u, 0, plane, work, sink, 4, 132);
  run<OP_RED_MAX_HINT, 4>("120 MB", n, 30000000u, 0, plane, work, sink, 4, 132);
  run<OP_RED_MAX_HINT, 4>("240 MB", n, big, 0, plane, work, sink, 4, 132);
  run<OP_RED_MAX, 4>("240 MB, no hint", n, big, 0, plane, work, sink, 4, 132);
  printf("## locality (RED.MAX evict_last, 40 MB plane): targets within a window around the sender's own index\n");
  run<OP_RED_MAX_HINT, 4>("window 1 MB (256 K words)", n, n, 262144u, plane, work, sink, 4, 132);
  run<OP_RED_MAX_HINT, 4>("window 64 KB (16 K words)", n, n, 16384u, plane, work, sink, 4, 132);
  run<OP_RED_MAX_HINT, 4>("window 4 KB (1 K words)", n, n, 1024u, plane, work, sink, 4, 132);
  printf("## ops per node (RED.MAX evict_last, 40 MB plane)\n");
  run<OP_RED_MAX_HINT, 1>("1 per node", n, n, 0, plane, work, sink, 4, 132);
  run<OP_RED_MAX_HINT, 8>("8 per node", n, n, 0, plane, work, sink, 4, 132);
  return 0;
}
