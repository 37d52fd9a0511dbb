// grow.cuh -- the one "grow a buffer" helper of the host code (BA handle, svs_chol6)
#pragma once
#include <cuda_runtime.h>

#include <cstddef>

namespace svs {

// Grows a device buffer and/or its pinned host twin (either may be null; both share `cap`) to hold at least n
// elements, with 25 % headroom so that a slowly growing window does not reallocate on every call.  The contents
// are not kept.  Only the buffers passed in are touched.
template <typename T>
cudaError_t grow(size_t n, size_t* cap, T** dev, T** pinned = nullptr) {
  if (n <= *cap) return cudaSuccess;
  if (dev && *dev) cudaFree(*dev);
  if (pinned && *pinned) cudaFreeHost(*pinned);
  if (dev) *dev = nullptr;
  if (pinned) *pinned = nullptr;
  *cap = 0;
  const size_t want = n + n / 4;
  cudaError_t e = dev ? cudaMalloc((void**)dev, want * sizeof(T)) : cudaSuccess;
  if (e == cudaSuccess && pinned) e = cudaMallocHost((void**)pinned, want * sizeof(T));
  if (e == cudaSuccess) *cap = want;
  return e;
}

}  // namespace svs
