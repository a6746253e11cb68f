// Host-side helpers of every translation unit of the library.  The error text behind nb_last_error (one thread-local buffer) and the
// launch counter behind nb_launch_count are defined once, in pan_api.cu.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <memory>

#include "../../include/neupan_b200.h"

namespace nb {

// formats the text nb_last_error returns and hands back `code`
int fail(int code, const char* fmt, ...);

// kernels the library has launched (nb_launch_count); every launch site adds its own
extern long long launches;

// device allocations alive in the process (nb_buffer_count): every DeviceArray allocation adds one, its free takes it away
inline std::atomic<int64_t> live_buffers{0};

// Owners of the library's device memory, streams and events.  Every cudaMalloc / cudaFree / cudaStreamDestroy / cudaEventDestroy of
// the library is here.  A handle frees its members with its own device current: destroy and the set calls select it first.
struct CudaFree {
  void operator()(void* p) const {
    cudaFree(p);
    --live_buffers;
  }
};
template <typename T>
using DeviceArray = std::unique_ptr<T[], CudaFree>;

// Frees what `a` holds, then allocates n (at least 1) elements into it: a regrowth never holds the old and the new buffer at once.
// On failure `a` is left empty, and the error is returned and cleared, so that it does not resurface at a later cudaGetLastError.
template <typename T>
cudaError_t alloc(DeviceArray<T>& a, size_t n) {
  a.reset();
  T* p = nullptr;
  const cudaError_t e = cudaMalloc((void**)&p, (n ? n : 1) * sizeof(T));
  if (e != cudaSuccess) {
    cudaGetLastError();
    return e;
  }
  ++live_buffers;
  a.reset(p);
  return e;
}

struct StreamDestroy {
  void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
};
struct EventDestroy {
  void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
};
using Stream = std::unique_ptr<CUstream_st, StreamDestroy>;
using Event = std::unique_ptr<CUevent_st, EventDestroy>;

// a non-blocking stream / an event without timing, created into an empty owner
inline cudaError_t create(Stream& s) {
  cudaStream_t q = nullptr;
  const cudaError_t e = cudaStreamCreateWithFlags(&q, cudaStreamNonBlocking);
  if (e == cudaSuccess) s.reset(q);
  return e;
}
inline cudaError_t create(Event& ev) {
  cudaEvent_t q = nullptr;
  const cudaError_t e = cudaEventCreateWithFlags(&q, cudaEventDisableTiming);
  if (e == cudaSuccess) ev.reset(q);
  return e;
}

}  // namespace nb

#define NB_CUDA(call)                                                                                 \
  do {                                                                                                \
    cudaError_t e__ = (call);                                                                         \
    if (e__ != cudaSuccess) return nb::fail(NB_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(e__)); \
  } while (0)
