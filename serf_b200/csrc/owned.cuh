// owned.cuh — the owners of a handle's device memory, mapped host words, streams, events and IPC mappings (host code only).
// Each owner releases what it holds in its destructor and is move-only.  A failed allocation leaves the owner as it was: the
// new resource is made first, then swapped in.
#pragma once
#include <cuda_runtime.h>

#include <cstring>
#include <string>
#include <utility>

#include "../../include/serfsim.h"

namespace sfs {

int serfsim_fail(int code, const char* msg);          // serfsim.cu: sets serfsim_last_error

// The one mapping of a CUDA error to a serfsim code: an allocation failure is SERFSIM_E_NOMEM, any other error SERFSIM_E_CUDA.
#define CU(call)                                                                                                 \
  do {                                                                                                           \
    const cudaError_t e_ = (call);                                                                               \
    if (e_ != cudaSuccess)                                                                                       \
      return sfs::serfsim_fail(e_ == cudaErrorMemoryAllocation ? SERFSIM_E_NOMEM : SERFSIM_E_CUDA,               \
                               (std::string(#call) + ": " + cudaGetErrorString(e_)).c_str());                    \
  } while (0)

// n elements of T in device memory.  It converts to T*, so launches and parameter blocks take it as they took the pointer.
template <class T>
class DevArray {
 public:
  DevArray() = default;
  DevArray(DevArray&& o) noexcept { *this = std::move(o); }
  DevArray& operator=(DevArray&& o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); return *this; }
  ~DevArray() { if (p_) cudaFree(p_); }

  cudaError_t alloc(size_t n) {                       // n elements, contents undefined
    DevArray a;
    const cudaError_t e = cudaMalloc(&a.p_, n * sizeof(T));
    if (!e) { a.n_ = n; *this = std::move(a); }
    return e;
  }
  cudaError_t grow(size_t n, cudaStream_t st) {       // n elements: the current ones copied over, the rest zero
    DevArray a;
    cudaError_t e = a.alloc(n);
    if (!e) e = a.fill(0, st);
    if (!e && p_) e = cudaMemcpyAsync(a.p_, p_, bytes(), cudaMemcpyDeviceToDevice, st);
    if (!e && p_) e = cudaStreamSynchronize(st);
    if (!e) *this = std::move(a);
    return e;
  }
  cudaError_t fill(int byte, cudaStream_t st) const { return n_ ? cudaMemsetAsync(p_, byte, bytes(), st) : cudaSuccess; }

  T* get() const { return p_; }
  operator T*() const { return p_; }
  size_t size() const { return n_; }
  size_t bytes() const { return n_ * sizeof(T); }

 private:
  T* p_ = nullptr;
  size_t n_ = 0;
};

// A CUDA object H made by Make(&h, args...) and released by Release(h).
template <class H, auto Make, auto Release>
class Owned {
 public:
  Owned() = default;
  Owned(Owned&& o) noexcept { *this = std::move(o); }
  Owned& operator=(Owned&& o) noexcept { std::swap(h_, o.h_); return *this; }
  ~Owned() { if (h_) Release(h_); }

  template <class... A>
  cudaError_t create(A... args) {
    Owned o;
    const cudaError_t e = Make(&o.h_, args...);
    if (!e) *this = std::move(o);
    return e;
  }
  operator H() const { return h_; }

 private:
  H h_{};
};

inline cudaError_t make_event(cudaEvent_t* e) { return cudaEventCreate(e); }
inline cudaError_t make_stream(cudaStream_t* s) { return cudaStreamCreateWithFlags(s, cudaStreamNonBlocking); }
inline cudaError_t open_ipc(void** p, cudaIpcMemHandle_t h) { return cudaIpcOpenMemHandle(p, h, cudaIpcMemLazyEnablePeerAccess); }
inline cudaError_t map_words(uint32_t** p, size_t n) {         // zeroed host words the device addresses directly
  const cudaError_t e = cudaHostAlloc(p, n * sizeof(uint32_t), cudaHostAllocMapped);
  if (!e) memset(*p, 0, n * sizeof(uint32_t));
  return e;
}
using Event = Owned<cudaEvent_t, make_event, cudaEventDestroy>;
using Stream = Owned<cudaStream_t, make_stream, cudaStreamDestroy>;
using IpcMapping = Owned<void*, open_ipc, cudaIpcCloseMemHandle>;      // a peer's exported buffer mapped into this process
using MappedWords = Owned<uint32_t*, map_words, cudaFreeHost>;         // kernels write them, the host reads them without a copy

}  // namespace sfs
