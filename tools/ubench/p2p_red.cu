// Micro-benchmark behind the choice of the cross-shard exchange (DESIGN §7): what does one H100 sustain towards a PEER
// GPU over NVLink for (a) scattered 4-byte RED.MAX into the peer's inbox plane (the "direct" exchange: no staging, no
// drain kernel), (b) scattered plain 4-byte stores, (c) coalesced 8-byte window entries (the window + drain exchange),
// (d) scattered byte stores (tile flags) — next to (e) the same scattered RED.MAX into LOCAL memory.  Both directions
// run at once (each GPU targets the other), like a sharded tick.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/ubench/p2p_red tools/ubench/p2p_red.cu
//   tools/ubench/p2p_red                 (on a machine with two GPUs)
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

typedef uint32_t u32;
typedef uint64_t u64;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

__device__ __forceinline__ u32 mix(u32 x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }

// MODE 0: scattered red.max.u32 (gpu scope)   1: scattered red.max.u32 (sys scope)   2: scattered st.u32
//      3: coalesced st.u64 (window entries)   4: scattered st.u8                      5: scattered atom.max with return (sys)
template <int MODE>
__global__ void __launch_bounds__(256, 4) k(u32 n_msgs, u32 n_dst, u32* dst, u64* win, unsigned char* bytes, u32 salt, u32* sink) {
  u32 acc = 0;
  for (u32 i = blockIdx.x * 256 + threadIdx.x; i < n_msgs; i += gridDim.x * 256) {
    const u32 t = mix(i ^ salt) % n_dst;
    if (MODE == 0) asm volatile("red.relaxed.gpu.global.max.u32 [%0], %1;" :: "l"(dst + t), "r"(i + 1) : "memory");
    if (MODE == 1) asm volatile("red.relaxed.sys.global.max.u32 [%0], %1;" :: "l"(dst + t), "r"(i + 1) : "memory");
    if (MODE == 2) dst[t] = i + 1;
    if (MODE == 3) win[i] = ((u64)(i + 1) << 32) | t;
    if (MODE == 4) bytes[t >> 8] = 1;
    if (MODE == 5) { u32 o; asm volatile("atom.relaxed.sys.global.max.u32 %0, [%1], %2;" : "=r"(o) : "l"(dst + t), "r"(i + 1) : "memory"); acc += o; }
  }
  if (acc == 0xdeadbeefu) *sink = acc;
}

struct Dev { u32* plane; u64* win; unsigned char* bytes; u32* sink; cudaStream_t st; cudaEvent_t a, b; };

template <int MODE>
static void run(const char* name, Dev* d, int ndev, bool remote, u32 n_msgs, u32 n_dst) {
  const int grid = 132 * 4, reps = 10;
  for (int phase = 0; phase < 2; ++phase) {          // phase 0 warm-up, phase 1 timed
    for (int g = 0; g < ndev; ++g) {
      CK(cudaSetDevice(g));
      const int tgt = remote ? (g + 1) % ndev : g;
      if (phase) CK(cudaEventRecord(d[g].a, d[g].st));
      for (int r = 0; r < (phase ? reps : 2); ++r)
        k<MODE><<<grid, 256, 0, d[g].st>>>(n_msgs, n_dst, d[tgt].plane, d[tgt].win, d[tgt].bytes, 7 * r + g + 100 * phase, d[g].sink);
      if (phase) CK(cudaEventRecord(d[g].b, d[g].st));
    }
    for (int g = 0; g < ndev; ++g) { CK(cudaSetDevice(g)); CK(cudaStreamSynchronize(d[g].st)); }
  }
  float worst = 0;
  for (int g = 0; g < ndev; ++g) { float ms; CK(cudaEventElapsedTime(&ms, d[g].a, d[g].b)); if (ms > worst) worst = ms; }
  const double us = 1e3 * worst / reps;
  printf("%-58s %9.1f us/pass  %7.1f Mmsg/s per GPU  %6.3f ns/msg\n", name, us, n_msgs / us, 1e3 * us / n_msgs);
  fflush(stdout);
}

int main(int argc, char** argv) {
  int ndev = 0;
  CK(cudaGetDeviceCount(&ndev));
  if (ndev < 2) { printf("needs 2 GPUs (found %d)\n", ndev); return 0; }
  ndev = 2;
  const u32 n_dst = argc > 1 ? (u32)atoll(argv[1]) : 5000000u;      // nodes of the target shard (plane = 4 B each)
  const u32 n_msgs = argc > 2 ? (u32)atoll(argv[2]) : 10000000u;     // cross-shard messages per pass (a plateau tick at world 2)
  Dev d[2];
  for (int g = 0; g < ndev; ++g) {
    CK(cudaSetDevice(g));
    int can = 0;
    CK(cudaDeviceCanAccessPeer(&can, g, (g + 1) % ndev));
    if (!can) { printf("no peer access %d -> %d\n", g, (g + 1) % ndev); return 0; }
    CK(cudaDeviceEnablePeerAccess((g + 1) % ndev, 0));
    CK(cudaMalloc(&d[g].plane, (size_t)n_dst * 4)); CK(cudaMalloc(&d[g].win, (size_t)n_msgs * 8));
    CK(cudaMalloc(&d[g].bytes, (n_dst >> 8) + 1)); CK(cudaMalloc(&d[g].sink, 4));
    CK(cudaMemset(d[g].plane, 0, (size_t)n_dst * 4));
    CK(cudaStreamCreate(&d[g].st)); CK(cudaEventCreate(&d[g].a)); CK(cudaEventCreate(&d[g].b));
  }
  printf("# %u messages per pass and GPU into a %u-node plane, both directions at once, 256 threads x 4 CTAs/SM\n", n_msgs, n_dst);
  run<0>("LOCAL  scattered red.max.u32 (gpu scope)", d, ndev, false, n_msgs, n_dst);
  run<0>("REMOTE scattered red.max.u32 (gpu scope)", d, ndev, true, n_msgs, n_dst);
  run<1>("REMOTE scattered red.max.u32 (sys scope)", d, ndev, true, n_msgs, n_dst);
  run<5>("REMOTE scattered atom.max.u32 with return (sys scope)", d, ndev, true, n_msgs / 8, n_dst);
  run<2>("REMOTE scattered st.u32", d, ndev, true, n_msgs, n_dst);
  run<3>("REMOTE coalesced st.u64 (window entries)", d, ndev, true, n_msgs, n_dst);
  run<3>("LOCAL  coalesced st.u64 (window entries)", d, ndev, false, n_msgs, n_dst);
  run<4>("REMOTE scattered st.u8 (tile flags)", d, ndev, true, n_msgs, n_dst);
  // smaller planes (world 8: 1.25 M-node shards, 0.55 M messages per peer and tick)
  run<0>("REMOTE scattered red.max.u32, 1.25 M-node plane, 4.4 M msgs", d, ndev, true, 4400000u, 1250000u);
  run<3>("REMOTE coalesced st.u64, 4.4 M msgs", d, ndev, true, 4400000u, 1250000u);
  return 0;
}
