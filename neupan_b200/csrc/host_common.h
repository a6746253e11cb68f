// Host-side helpers of every translation unit of the library.  The error text behind nb_last_error (one thread-local buffer) and the
// launch counter behind nb_launch_count are defined once, in pan_api.cu.
#pragma once
#include <cuda_runtime.h>

#include "../../include/neupan_b200.h"

namespace nb {

// formats the text nb_last_error returns and hands back `code`
int fail(int code, const char* fmt, ...);

// kernels the library has launched (nb_launch_count); every launch site adds its own
extern long long launches;

template <typename T>
cudaError_t dalloc(T** p, size_t n) {
  return cudaMalloc((void**)p, (n ? n : 1) * sizeof(T));
}

}  // namespace nb

#define NB_CUDA(call)                                                                                 \
  do {                                                                                                \
    cudaError_t e__ = (call);                                                                         \
    if (e__ != cudaSuccess) return nb::fail(NB_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(e__)); \
  } while (0)
