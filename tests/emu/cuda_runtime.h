// tests/emu/cuda_runtime.h — a minimal CUDA-on-CPU shim, TEST INFRASTRUCTURE ONLY.
//
// Purpose: compile the product's own kernel and host sources (serf_b200/csrc/*.cu) with g++ and run them on a machine
// without a GPU, so that the LOGIC of the kernels (indexing, tile skipping, queue handling, counters, the C-ABI host
// code around them) can be compared with the oracle in the CPU test-suite.  It says nothing about performance, memory
// ordering, cache behaviour or PTX semantics — the GPU parity tests (-m gpu) remain the proof for the real build.
// Nothing under serf_b200/ includes or links this; the product library is built by nvcc from the same sources and
// fails with SERFSIM_E_NO_DEVICE without a GPU.
//
// Execution model (per rank; multi-rank runs give every rank its own OS thread and the engine state is thread-local,
// peer windows are plain shared host memory with real acquire/release on the flags): one CTA at a time; every CUDA thread of the CTA is a fiber on one OS thread; fibers
// switch only at collectives (__syncthreads, warp shuffles / votes), where they wait for the other lanes exactly like
// the hardware does.  __shared__ becomes `static` (CTAs run one after another).  Atomics are plain read-modify-writes.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <tuple>
#include <utility>

#ifndef SERFSIM_EMU
#error "tests/emu/cuda_runtime.h is only for -DSERFSIM_EMU host builds of the kernels"
#endif

// ---- language keywords ----
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __grid_constant__
#define __shared__ static thread_local              // one CTA at a time PER RANK THREAD (multi-rank runs: one OS thread per rank)
#define __align__(n) __attribute__((aligned(n)))

// ---- vector types ----
struct uint3 { unsigned x, y, z; };
struct uint4 { unsigned x, y, z, w; };
struct alignas(8) uint2 { unsigned x, y; };
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{x, y}; }

// ---- engine ----
namespace emu {
struct LaneCtx { uint3 tid, bid, bdim, gdim; };
extern thread_local LaneCtx* cur;
void run_grid(unsigned grid, unsigned block, const std::function<void()>& body);
void cta_barrier();
unsigned long long warp_exchange(unsigned long long v, int src_lane_xor, int src_lane_abs);   // returns the value of lane (abs >= 0 ? abs : lane ^ xor)
unsigned warp_ballot(bool pred);
unsigned warp_reduce_or(unsigned v);
unsigned lane_id();
void polite_wait(unsigned long spins);                          // yields the OS thread; aborts the process after ~120 s of fruitless polling (a peer rank died)
extern unsigned long probes[32];                              // coverage probes: SFS_PROBE(i) in the kernels, read by tests through emu_probe()

template <class F>
struct Bound {
  unsigned grid, block;
  F f;
  template <class... A>
  void operator()(A&&... a) {
    auto args = std::make_tuple(std::decay_t<A>(a)...);            // kernel arguments are passed by value, once per launch
    run_grid(grid, block, [&] { std::apply(f, args); });
  }
};
struct Launch {
  unsigned grid, block;
  template <class F> Bound<F> with(F f) const { return Bound<F>{grid, block, f}; }
};
}  // namespace emu

#define threadIdx (emu::cur->tid)
#define blockIdx (emu::cur->bid)
#define blockDim (emu::cur->bdim)
#define gridDim (emu::cur->gdim)
#define SFS_LAUNCH(grid, block, smem, stream, ...) \
  emu::Launch{(unsigned)(grid), (unsigned)(block)}.with([&](auto&&... a_) { __VA_ARGS__(a_...); })

// ---- device intrinsics ----
inline void __syncthreads() { emu::cta_barrier(); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::warp_ballot(false); }
inline unsigned __shfl_xor_sync(unsigned, unsigned v, int o) { return (unsigned)emu::warp_exchange(v, o, -1); }
inline int __shfl_xor_sync(unsigned, int v, int o) { return (int)emu::warp_exchange((unsigned)v, o, -1); }
inline unsigned long __shfl_xor_sync(unsigned, unsigned long v, int o) { return (unsigned long)emu::warp_exchange(v, o, -1); }
inline unsigned long long __shfl_xor_sync(unsigned, unsigned long long v, int o) { return emu::warp_exchange(v, o, -1); }
inline unsigned __shfl_sync(unsigned mask, unsigned v, int src) {
  if (mask == (1u << emu::lane_id())) return v;              // the single-lane groups __match_any_sync hands out above
  return (unsigned)emu::warp_exchange(v, 0, src & 31);
}
inline unsigned __ballot_sync(unsigned, int pred) { return emu::warp_ballot(pred != 0); }
inline int __any_sync(unsigned, int pred) { return emu::warp_ballot(pred != 0) != 0; }
inline unsigned __reduce_or_sync(unsigned, unsigned v) { return emu::warp_reduce_or(v); }
// Divergent-context helpers (only the cross-shard staging uses them): every lane acts as its own leader, which is a
// valid outcome of warp aggregation.
inline unsigned __activemask() { return 1u << emu::lane_id(); }
inline unsigned __match_any_sync(unsigned, unsigned) { return 1u << emu::lane_id(); }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __ffs(int v) { return __builtin_ffs(v); }
template <class T> inline T __ldg(const T* p) { emu::probes[15] += sizeof(T); return *p; }   // read-only-path loads (row offsets, neighbour gathers)
template <class T> inline T __ldcg(const T* p) { return *p; }
inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
inline void __threadfence_system() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p = o + v; return o; }
inline int atomicAdd(int* p, int v) { int o = *p; *p = o + v; return o; }
inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; *p = o + v; return o; }
inline unsigned atomicMax(unsigned* p, unsigned v) { unsigned o = *p; if (v > o) *p = v; return o; }
inline unsigned long long atomicMax(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; if (v > o) *p = v; return o; }
inline unsigned atomicMin(unsigned* p, unsigned v) { unsigned o = *p; if (v < o) *p = v; return o; }
inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; if (v < o) *p = v; return o; }
inline unsigned atomicOr(unsigned* p, unsigned v) { unsigned o = *p; *p = o | v; return o; }
template <class T> inline T min(T a, T b) { return b < a ? b : a; }
template <class T> inline T max(T a, T b) { return a < b ? b : a; }
inline unsigned long min(unsigned long a, unsigned long long b) { return b < a ? (unsigned long)b : a; }

// ---- runtime API (host side): device memory is host memory, streams are in-order by construction ----
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorNotSupported = 801 };
typedef struct emuStream_st* cudaStream_t;
typedef struct emuEvent_st* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
enum { cudaStreamNonBlocking = 1 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16, cudaDevAttrComputeCapabilityMajor = 75, cudaDevAttrComputeCapabilityMinor = 76, cudaDevAttrMaxPersistingL2CacheSize = 108, cudaDevAttrMaxAccessPolicyWindowSize = 109 };
enum cudaLimit { cudaLimitPersistingL2CacheSize = 6 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum cudaAccessProperty { cudaAccessPropertyNormal = 0, cudaAccessPropertyStreaming = 1, cudaAccessPropertyPersisting = 2 };
enum cudaStreamAttrID { cudaStreamAttributeAccessPolicyWindow = 1 };
struct cudaAccessPolicyWindow { void* base_ptr; size_t num_bytes; float hitRatio; cudaAccessProperty hitProp, missProp; };
union cudaStreamAttrValue { cudaAccessPolicyWindow accessPolicyWindow; int pad; };
struct cudaIpcMemHandle_t { char reserved[64]; };
enum { cudaIpcMemLazyEnablePeerAccess = 1 };

template <class T> inline cudaError_t cudaMalloc(T** p, size_t n) {
  void* q = nullptr;
  if (posix_memalign(&q, 256, n ? ((n + 255) / 256) * 256 : 256)) return cudaErrorMemoryAllocation;
  memset(q, 0xA5, n);                                        // like the device: fresh memory is NOT zero
  *p = (T*)q;
  return cudaSuccess;
}
inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
template <class T> inline cudaError_t cudaMallocHost(T** p, size_t n) { *p = (T*)malloc(n ? n : 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
constexpr unsigned cudaHostAllocMapped = 2;
template <class T> inline cudaError_t cudaHostAlloc(T** p, size_t n, unsigned) { *p = (T*)malloc(n ? n : 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
template <class T> inline cudaError_t cudaHostGetDevicePointer(T** d, void* h, unsigned) { *d = (T*)h; return cudaSuccess; }
inline cudaError_t cudaMemset(void* p, int v, size_t n) { memset(p, v, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (cudaStream_t)malloc(8); return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamSetAttribute(cudaStream_t, cudaStreamAttrID, const cudaStreamAttrValue*) { return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = (cudaEvent_t)malloc(8); return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.001f; return cudaSuccess; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated CUDA error"; }
inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr a, int) {
  switch (a) {
    case cudaDevAttrMultiProcessorCount: { const char* e = getenv("SERFSIM_EMU_SMS"); *v = e ? atoi(e) : 1; break; }
    case cudaDevAttrComputeCapabilityMajor: *v = 9; break;          // minor: 0 (default)
    default: *v = 0;
  }
  return cudaSuccess;
}
inline cudaError_t cudaDeviceSetLimit(cudaLimit, size_t) { return cudaSuccess; }
template <class F> inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
// "IPC" between ranks that are threads of one process: the handle is the pointer itself
inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p) { memset(h, 0, sizeof(*h)); memcpy(h->reserved, &p, sizeof(p)); return cudaSuccess; }
inline cudaError_t cudaIpcOpenMemHandle(void** out, cudaIpcMemHandle_t h, unsigned) { memcpy(out, h.reserved, sizeof(*out)); return cudaSuccess; }
inline cudaError_t cudaIpcCloseMemHandle(void*) { return cudaSuccess; }
