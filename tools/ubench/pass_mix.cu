// Where does a saturated pass's time go: the L2 policy of its streams, or the round trip of the RED filter?  One kernel reproduces the
// access mix of a saturated per-view pass of the single-slot tick kernel, one thread per node, 3 CTAs of 256 threads per SM (its cap):
//   record (32 B, two 128-bit evict_first / no-L1-allocate loads), node word (8 B load + store), queue word (4 B load + store),
//   4 picks out of the node's 16-entry CSR row, and per kind in flight 4 peeks of the destination words plus RED.MAX (evict_last)
//   of the ones below the value — every sender sends the same value, as in a wave, so about one RED per node and kind is issued.
// Variants:
//   policy   today: queue word plain, CSR gather __ldg (the tick kernel's accesses) | first: both carry evict_first
//   gather   ldg: __ldg | ef-l1: evict_first, allocated in L1 | ef-na: evict_first, not allocated in L1
//   send     serial: per kind, peek its 4 words, wait, RED (the tick kernel) | together: peek every kind's words, then the REDs
//            | deferred: enqueue (word, value) in shared memory, fetch the 16-byte group of each word with cp.async.cg (L2 only),
//              decide the REDs after the NEXT node's loads have returned
// Results in DESIGN §5 ("Every plane of a pass carries an L2 policy").
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -Xptxas -v -o tools/ubench/pass_mix tools/ubench/pass_mix.cu
//   tools/ubench/pass_mix [n]           (on the GPU)
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

typedef uint32_t u32;
typedef uint64_t u64;

__device__ __forceinline__ u32 mix(u32 x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }
__device__ __forceinline__ u64 pol_last() { u64 p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ u64 pol_first() { u64 p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }

enum { POL_TODAY = 0, POL_FIRST = 1 };
enum { COL_LDG = 0, COL_EF_L1 = 1, COL_EF_NA = 2 };
enum { SEND_SERIAL = 0, SEND_TOGETHER = 1, SEND_DEFERRED = 2 };
constexpr int FAN = 4, DEG = 16, KMAX = 2, QCAP = FAN * KMAX;
constexpr u32 VAL = 0x1234u;

__device__ __forceinline__ u32 ld_col(const u32* p, u64 pf, int col) {
  u32 v;
  if (col == COL_LDG) v = __ldg(p);
  else if (col == COL_EF_L1) asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pf));
  else asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pf));
  return v;
}
__device__ __forceinline__ u32 ld_u32_ef(const u32* p, u64 pf) { u32 v; asm volatile("ld.global.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pf)); return v; }
__device__ __forceinline__ void st_u32_ef(u32* p, u32 v, u64 pf) { asm volatile("st.global.L2::cache_hint.u32 [%0], %1, %2;" :: "l"(p), "r"(v), "l"(pf) : "memory"); }
__device__ __forceinline__ u32 peek(const u32* p, u64 pl) { u32 v; asm volatile("ld.global.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pl)); return v; }
__device__ __forceinline__ void red_max(u32* p, u32 v, u64 pl) { asm volatile("red.relaxed.gpu.global.max.L2::cache_hint.u32 [%0], %1, %2;" :: "l"(p), "r"(v), "l"(pl) : "memory"); }

template <int POL, int COL, int SEND, int K>
__global__ void __launch_bounds__(256, 3) pass_mix(const uint4* rec, u64* node, u32* qword, const u32* col, u32* plane, u32 n, u32 salt) {
  __shared__ __align__(16) uint4 fetch_s[SEND == SEND_DEFERRED ? QCAP * 256 : 1];   // entry e of thread t at e·256 + t
  __shared__ u32 off_s[SEND == SEND_DEFERRED ? QCAP * 256 : 1];
  const u64 pf = pol_first(), pl = pol_last();
  u32 queued = 0;
  auto drain = [&]() {
    asm volatile("cp.async.wait_all;" ::: "memory");
    for (u32 e = 0; e < queued; ++e) {
      const u32 o = off_s[e * 256 + threadIdx.x];
      const uint4 g = fetch_s[e * 256 + threadIdx.x];
      const u32 w = (o & 3) == 0 ? g.x : (o & 3) == 1 ? g.y : (o & 3) == 2 ? g.z : g.w;
      if (w < VAL) red_max(plane + o, VAL, pl);
    }
    queued = 0;
  };
  for (u32 v = blockIdx.x * 256 + threadIdx.x; v < n; v += gridDim.x * 256) {
    uint4 a, b;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%8], %9;\n\t"
                 "ld.global.L1::no_allocate.L2::cache_hint.v4.u32 {%4,%5,%6,%7}, [%8+16], %9;"
                 : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w), "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w) : "l"(rec + 2 * (size_t)v), "l"(pf));
    u64 ns;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(ns) : "l"(node + v), "l"(pf));
    const u32 q = POL == POL_FIRST ? ld_u32_ef(qword + v, pf) : qword[v];
    const u32 h = mix(v ^ salt);
    u32 tg[FAN];
#pragma unroll
    for (int j = 0; j < FAN; ++j) tg[j] = ld_col(col + (size_t)v * DEG + (mix(h + j) & (DEG - 1)), pf, COL);
    // the node logic: the record and the node word feed the stores, so every load has returned before them
    const u32 x = a.x ^ a.y ^ a.z ^ a.w ^ b.x ^ b.y ^ b.z ^ b.w;
    asm volatile("st.global.L2::cache_hint.u64 [%0], %1, %2;" :: "l"(node + v), "l"(ns + x), "l"(pf) : "memory");
    if (POL == POL_FIRST) st_u32_ef(qword + v, q + 1, pf); else qword[v] = q + 1;
    if (SEND == SEND_DEFERRED) {
      if (queued) drain();                                 // the previous node's words were fetched while this node's loads were in flight
#pragma unroll
      for (int k = 0; k < K; ++k)
#pragma unroll
        for (int j = 0; j < FAN; ++j) {
          const u32 o = k * n + tg[j], e = k * FAN + j;
          off_s[e * 256 + threadIdx.x] = o;
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"((u32)__cvta_generic_to_shared(&fetch_s[e * 256 + threadIdx.x])), "l"(plane + (o & ~3u)) : "memory");
        }
      asm volatile("cp.async.commit_group;" ::: "memory");
      queued = K * FAN;
    } else if (SEND == SEND_TOGETHER) {
      u32 held[K][FAN];
#pragma unroll
      for (int k = 0; k < K; ++k)
#pragma unroll
        for (int j = 0; j < FAN; ++j) held[k][j] = peek(plane + k * n + tg[j], pl);
#pragma unroll
      for (int k = 0; k < K; ++k)
#pragma unroll
        for (int j = 0; j < FAN; ++j) if (held[k][j] < VAL) red_max(plane + k * n + tg[j], VAL, pl);
    } else {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        u32 held[FAN];
#pragma unroll
        for (int j = 0; j < FAN; ++j) held[j] = peek(plane + k * n + tg[j], pl);
#pragma unroll
        for (int j = 0; j < FAN; ++j) if (held[j] < VAL) red_max(plane + k * n + tg[j], VAL, pl);
      }
    }
  }
  if (SEND == SEND_DEFERRED && queued) drain();
}

__global__ void init_col(u32* col, size_t m, u32 n) {
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < m; i += (size_t)gridDim.x * 256) col[i] = __umulhi(mix((u32)i * 2654435761u + 12345u), n);
}

static void check(cudaError_t e, const char* what) { if (e != cudaSuccess) { printf("CUDA error %s: %s\n", what, cudaGetErrorString(e)); exit(1); } }

struct Ctx { u32 n; uint4* rec; u64* node; u32 *qword, *col, *plane; cudaEvent_t a, b; };
typedef void (*Kern)(const uint4*, u64*, u32*, const u32*, u32*, u32, u32);

// Mean and best over reps of one launch (ms); the planes start at zero, as at the beginning of a pass.
static void timed(Ctx& c, Kern k, int K, double& mean, double& best) {
  const int reps = 10;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  mean = 0; best = 1e30;
  for (int r = 0; r < reps + 2; ++r) {
    check(cudaMemset(c.plane, 0, (size_t)c.n * 4 * K), "memset plane");
    check(cudaEventRecord(c.a), "record");
    k<<<sms * 3, 256>>>(c.rec, c.node, c.qword, c.col, c.plane, c.n, 77 + r);
    check(cudaEventRecord(c.b), "record");
    check(cudaEventSynchronize(c.b), "sync");
    float ms = 0;
    cudaEventElapsedTime(&ms, c.a, c.b);
    if (r >= 2) { mean += ms / reps; if (ms < best) best = ms; }
  }
  check(cudaGetLastError(), "launch");
}

struct Variant { const char* name; Kern k1, k2; };
#define V(name, POL, COL, SEND) {name, pass_mix<POL, COL, SEND, 1>, pass_mix<POL, COL, SEND, 2>}

int main(int argc, char** argv) {
  Ctx c;
  c.n = argc > 1 ? (u32)atoll(argv[1]) : 10000000u;
  const size_t m = (size_t)c.n * DEG;
  check(cudaMalloc(&c.rec, (size_t)c.n * 32), "malloc");
  check(cudaMalloc(&c.node, (size_t)c.n * 8), "malloc");
  check(cudaMalloc(&c.qword, (size_t)c.n * 4), "malloc");
  check(cudaMalloc(&c.col, m * 4), "malloc");
  check(cudaMalloc(&c.plane, (size_t)c.n * 4 * KMAX), "malloc");
  check(cudaMemset(c.rec, 1, (size_t)c.n * 32), "memset");
  check(cudaMemset(c.node, 0, (size_t)c.n * 8), "memset");
  check(cudaMemset(c.qword, 0, (size_t)c.n * 4), "memset");
  init_col<<<1024, 256>>>(c.col, m, c.n);
  check(cudaDeviceSynchronize(), "init");
  cudaEventCreate(&c.a); cudaEventCreate(&c.b);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  printf("# %s, %u nodes, %d deliveries per node and kind, CSR %.0f MB, plane %.0f MB per kind\n", prop.name, c.n, FAN, m * 4 / 1e6, c.n * 4 / 1e6);
  // the first variant runs again last: the spread between its two runs is the noise the others are read against
  const Variant vs[] = {
      V("(a)  today: qword plain, gather ldg, serial", POL_TODAY, COL_LDG, SEND_SERIAL),
      V("(b1) evict_first, gather ef + L1", POL_FIRST, COL_EF_L1, SEND_SERIAL),
      V("(b2) evict_first, gather ef no-L1", POL_FIRST, COL_EF_NA, SEND_SERIAL),
      V("(c)  today, peeks together", POL_TODAY, COL_LDG, SEND_TOGETHER),
      V("(c1) b1 + peeks together", POL_FIRST, COL_EF_L1, SEND_TOGETHER),
      V("(d)  today, deferred (cp.async.cg)", POL_TODAY, COL_LDG, SEND_DEFERRED),
      V("(d1) b1 + deferred", POL_FIRST, COL_EF_L1, SEND_DEFERRED),
      V("(a)  again", POL_TODAY, COL_LDG, SEND_SERIAL),
  };
  for (const Variant& v : vs) {
    double m1, b1, m2, b2;
    timed(c, v.k1, 1, m1, b1);
    timed(c, v.k2, 2, m2, b2);
    printf("%-44s 1 kind %8.1f us (best %8.1f) %6.1f G deliveries/s | 2 kinds %8.1f us (best %8.1f) %6.1f G/s\n", v.name, 1e3 * m1, 1e3 * b1,
           (double)c.n * FAN / (m1 * 1e-3) / 1e9, 1e3 * m2, 1e3 * b2, 2.0 * c.n * FAN / (m2 * 1e-3) / 1e9);
  }
  return 0;
}
