// handle.cuh -- the host plumbing every opaque handle of the C ABI shares: its device, stream and error text, the CUDA
// check, opening and closing the handle on its device, the "grow a buffer" helper and the layout of a buffer
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstddef>
#include <string>

#include "../../include/svs_b200.h"

namespace svs {

// The head of every handle (struct svs_x : svs::Handle).  The stream, when the handle has one, ends with the handle.
struct Handle {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  ~Handle() {
    if (stream) cudaStreamDestroy(stream);
  }
};

// On a failed CUDA call: the call's text and CUDA's error string become h's error, the entry point returns SVS_ERR_CUDA.
#define SVS_CK(h, call)                                                 \
  do {                                                                  \
    cudaError_t e_ = (call);                                            \
    if (e_ != cudaSuccess) {                                            \
      (h)->err = std::string(#call) + ": " + cudaGetErrorString(e_);    \
      return SVS_ERR_CUDA;                                              \
    }                                                                   \
  } while (0)

inline int fail(Handle* h, int code, const std::string& msg) {
  h->err = msg;
  return code;
}

// The device part of a create: SVS_ERR_NOGPU without a CUDA device; device < 0 becomes the current device, which is
// made h's device and current; then h's non-blocking stream (SVS_ERR_CUDA when either fails).  stream = false
// (svs_chol6, which works on its internal BA handle's stream): no stream, and a device past the last one is
// SVS_ERR_INVALID.
inline int open_handle(Handle* h, int& device, bool stream = true) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return SVS_ERR_NOGPU;
  if (device < 0) cudaGetDevice(&device);
  if (!stream && device >= n) return SVS_ERR_INVALID;
  h->device = device;
  if (cudaSetDevice(device) != cudaSuccess) return SVS_ERR_CUDA;
  if (stream && cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) return SVS_ERR_CUDA;
  return SVS_OK;
}

// The start of a destroy: the handle's device becomes current and its stream drains.  The module frees its buffers
// after this; `delete` then ends the stream.
inline void begin_close(Handle* h) {
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
}

inline const char* last_error(const Handle* h) { return h ? h->err.c_str() : "null handle"; }

// true when p is device (or managed) memory of `device`; a failed query leaves no sticky error behind
inline bool on_device(int device, const void* p) {
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == device;
}

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

// Lays a module's arrays out in one buffer, each 256-byte aligned, in take order; n = 0 still gets a slot.  A pass
// with base == nullptr only sizes (every take returns nullptr): off is then the bytes the buffer needs.  The idiom is
// a sizing pass, grow to `off`, then the same takes on the buffer.  `off` is also the mark of where the next take lies.
struct Bump {
  char* base; size_t off = 0;
  template <typename T> T* take(size_t n) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += ((std::max<size_t>(n, 1) * sizeof(T) + 255) / 256) * 256;
    return p;
  }
};

}  // namespace svs
