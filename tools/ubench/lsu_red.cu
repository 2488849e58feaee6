// Micro-benchmarks behind the "plateau ticks are LSU-issue bound" reading of DESIGN.md ("What comes next", item 4):
// how fast can one H100 issue (a) scattered RED.MAX into an L2-resident 40 MB plane, (b) scattered 4-byte gathers from a
// 640 MB array (4 picks inside a 64-byte row, like the neighbour picks), (c) both together, (d) the coalesced 32-byte
// record stream next to them — each at the tick kernel's occupancy (256 threads, 4 CTAs per SM).
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/ubench/lsu_red tools/ubench/lsu_red.cu   (cross-compiles here)
//   tools/ubench/lsu_red                 (on the GPU)
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

typedef uint32_t u32;
typedef uint64_t u64;

__device__ __forceinline__ u32 mix(u32 x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }
__device__ __forceinline__ u64 pol_last() { u64 p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ u64 pol_first() { u64 p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ void red_max(u32* ptr, u32 v, u64 pol) { asm volatile("red.relaxed.gpu.global.max.L2::cache_hint.u32 [%0], %1, %2;" :: "l"(ptr), "r"(v), "l"(pol) : "memory"); }

// mode bit 0: 4 scattered REDs per node, bit 1: 4 gathers inside the node's 64-byte row, bit 2: stream a 32-byte record per node
template <int MODE>
__global__ void __launch_bounds__(256, 4) k(u32 n, u32* plane, const u32* col, const uint4* rec, u32 salt, u32* sink) {
  const u64 pl = pol_last(), pf = pol_first();
  u32 acc = 0;
  for (u32 v = blockIdx.x * 256 + threadIdx.x; v < n; v += gridDim.x * 256) {
    u32 tg[4];
    const u32 h = mix(v ^ salt);
#pragma unroll
    for (int j = 0; j < 4; ++j) tg[j] = (MODE & 2) ? __ldg(col + (size_t)v * 16 + ((h >> (4 * j)) & 15)) : mix(h + j) % n;
    if (MODE & 4) {
      u32 w[8];
      asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%8], %9;\n\t"     // the record load of the tick kernel
                   "ld.global.L1::no_allocate.L2::cache_hint.v4.u32 {%4,%5,%6,%7}, [%8+16], %9;"
                   : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "l"(rec + 2 * (size_t)v), "l"(pf));
      acc += w[0] ^ w[7];
    }
    if (MODE & 1) {
#pragma unroll
      for (int j = 0; j < 4; ++j) red_max(plane + tg[j], v + 1, pl);
    } else {
      acc += tg[0] ^ tg[1] ^ tg[2] ^ tg[3];
    }
  }
  if (acc == 0xdeadbeefu) *sink = acc;
}

template <int MODE>
static void run(const char* name, u32 n, u32* plane, const u32* col, const uint4* rec, u32* sink) {
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  const int grid = 132 * 4;
  for (int w = 0; w < 3; ++w) k<MODE><<<grid, 256>>>(n, plane, col, rec, w, sink);
  cudaEventRecord(a);
  const int reps = 10;
  for (int r = 0; r < reps; ++r) k<MODE><<<grid, 256>>>(n, plane, col, rec, 100 + r, sink);
  cudaEventRecord(b);
  cudaEventSynchronize(b);
  float ms = 0;
  cudaEventElapsedTime(&ms, a, b);
  const double us = 1e3 * ms / reps;
  const double clk = 1.9e9;      // nominal; the per-lane figures below scale with the real SM clock
  const double lanes = (double)n / 132.0;                          // node-iterations per SM
  printf("%-44s %8.1f us/pass  %7.2f ns/node  ~%5.2f SM-cycles per node per SM\n", name, us, 1e3 * us / n, us * 1e-6 * clk / lanes);
  if (cudaGetLastError() != cudaSuccess) { printf("CUDA error\n"); exit(1); }
}

int main(int argc, char** argv) {
  const u32 n = argc > 1 ? (u32)atoll(argv[1]) : 10000000u;
  u32 *plane, *col, *sink; uint4* rec;
  cudaMalloc(&plane, (size_t)n * 4); cudaMalloc(&col, (size_t)n * 16 * 4); cudaMalloc(&rec, (size_t)n * 32); cudaMalloc(&sink, 4);
  cudaMemset(plane, 0, (size_t)n * 4); cudaMemset(rec, 1, (size_t)n * 32);
  u32* hcol = (u32*)malloc((size_t)n * 16 * 4);
  u64 s = 88172645463325252ull;
  for (size_t i = 0; i < (size_t)n * 16; ++i) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; hcol[i] = (u32)(s % n); }
  cudaMemcpy(col, hcol, (size_t)n * 16 * 4, cudaMemcpyHostToDevice);
  printf("# n = %u nodes, 256 threads x 4 CTAs/SM, 10 passes each (tick kernel plateau: ~390 us per pass of 10 M nodes)\n", n);
  run<1>("4 scattered RED.MAX / node (targets hashed)", n, plane, col, rec, sink);
  run<2>("4 gathers in own 64-B row / node", n, plane, col, rec, sink);
  run<3>("4 gathers + 4 RED.MAX / node", n, plane, col, rec, sink);
  run<4>("32-B record stream / node", n, plane, col, rec, sink);
  run<7>("record stream + 4 gathers + 4 RED.MAX / node", n, plane, col, rec, sink);
  return 0;
}
