// prep.cu -- per-frame image preprocessing on sm_90a (SURVEY.md 8f rank 2, a "next" row):
// FrameGrabber::preprocessing (scavislam/frame_grabber.cpp:287-336):
//   cv::buildPyramid(uint8)                       -> k_pyrdown_u8   (5x5 [1 4 6 4 1]/16, (s + 128) >> 8, reflect-101)
//   gpu_uint8.convertTo(CV_32F, 1/255)            -> k_u8_to_f32
//   cv::gpu::pyrDown(float)                       -> k_pyrdown_f32  (same taps, float, reflect-101)
//   createDerivFilter_GPU(dx|dy, ksize 1, REPLICATE) (frame_grabber.cpp:104-115) -> k_deriv ([-1 0 1])
// Pure streaming image work, HBM-bound at ~1 B/px in + 13 B/px out for level 0; every output stays
// on the device so that the FAST, dense-tracking and matcher handles can take it without a host trip.
// The arithmetic order follows OpenCV's CPU pyrDown (row pass 6*c + 4*(l+r) + ll + rr, column pass,
// then * 1/256) and is compiled without FMA contraction so that it can be checked against cv2.
#include <algorithm>
#include <cstring>
#include <string>

#include <cuda_runtime.h>

#include "../../include/svs_b200.h"
#include "handle.cuh"

namespace {

constexpr int kMaxLv = 8;

__device__ __forceinline__ int reflect101(int i, int n) {
  if (n == 1) return 0;
  while (i < 0 || i >= n) i = i < 0 ? -i : 2 * n - 2 - i;
  return i;
}

__global__ void k_u8_to_f32(const unsigned char* __restrict__ src, int spitch, float* __restrict__ dst, int dstride, int w, int h) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x < w && y < h) dst[(size_t)y * dstride + x] = (float)src[(size_t)y * spitch + x] * (1.f / 255.f);
}

// one output pixel per thread; dst is (w+1)/2 x (h+1)/2
__global__ void k_pyrdown_f32(const float* __restrict__ src, int sstride, int w, int h, float* __restrict__ dst, int dstride) {
  const int dw = (w + 1) / 2, dh = (h + 1) / 2;
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= dw || y >= dh) return;
  float rows[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const float* r = src + (size_t)reflect101(2 * y - 2 + k, h) * sstride;
    const float c = r[reflect101(2 * x, w)], l = r[reflect101(2 * x - 1, w)], rr = r[reflect101(2 * x + 1, w)];
    const float ll = r[reflect101(2 * x - 2, w)], r2 = r[reflect101(2 * x + 2, w)];
    rows[k] = c * 6.f + (l + rr) * 4.f + ll + r2;
  }
  dst[(size_t)y * dstride + x] = (rows[2] * 6.f + (rows[1] + rows[3]) * 4.f + rows[0] + rows[4]) * (1.f / 256.f);
}

__global__ void k_pyrdown_u8(const unsigned char* __restrict__ src, int spitch, int w, int h, unsigned char* __restrict__ dst, int dpitch) {
  const int dw = (w + 1) / 2, dh = (h + 1) / 2;
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= dw || y >= dh) return;
  int rows[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const unsigned char* r = src + (size_t)reflect101(2 * y - 2 + k, h) * spitch;
    rows[k] = r[reflect101(2 * x, w)] * 6 + (r[reflect101(2 * x - 1, w)] + r[reflect101(2 * x + 1, w)]) * 4 +
              r[reflect101(2 * x - 2, w)] + r[reflect101(2 * x + 2, w)];
  }
  dst[(size_t)y * dpitch + x] = (unsigned char)((rows[2] * 6 + (rows[1] + rows[3]) * 4 + rows[0] + rows[4] + 128) >> 8);
}

__global__ void k_deriv(const float* __restrict__ src, int stride, int w, int h, float* __restrict__ dx, float* __restrict__ dy) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const int xl = max(x - 1, 0), xr = min(x + 1, w - 1), yu = max(y - 1, 0), yd = min(y + 1, h - 1);
  dx[(size_t)y * stride + x] = src[(size_t)y * stride + xr] - src[(size_t)y * stride + xl];
  dy[(size_t)y * stride + x] = src[(size_t)yd * stride + x] - src[(size_t)yu * stride + x];
}

}  // namespace

struct svs_prep : svs::Handle {
  int nlevels = 0, w[kMaxLv] = {}, h[kMaxLv] = {}, pitch8[kMaxLv] = {}, stride32[kMaxLv] = {};
  unsigned char* u8[kMaxLv] = {};
  float* f32[kMaxLv][3] = {};   // image, dx, dy
  unsigned char* stage = nullptr;
};

extern "C" {

int svs_prep_create(int device, int w, int hgt, int nlevels, svs_prep** out) {
  if (!out || w <= 0 || hgt <= 0 || nlevels <= 0 || nlevels > kMaxLv) return SVS_ERR_INVALID;
  *out = nullptr;
  svs_prep* h = new svs_prep();
  if (int rc = svs::open_handle(h, device)) {
    delete h;
    return rc;
  }
  h->nlevels = nlevels;
  bool ok = true;
  for (int l = 0; ok && l < nlevels; ++l) {
    h->w[l] = l ? (h->w[l - 1] + 1) / 2 : w;
    h->h[l] = l ? (h->h[l - 1] + 1) / 2 : hgt;
    h->pitch8[l] = ((h->w[l] + 255) / 256) * 256;
    h->stride32[l] = ((h->w[l] + 63) / 64) * 64;
    ok = cudaMalloc(&h->u8[l], (size_t)h->pitch8[l] * h->h[l]) == cudaSuccess;
    for (int k = 0; ok && k < 3; ++k) ok = cudaMalloc(&h->f32[l][k], sizeof(float) * (size_t)h->stride32[l] * h->h[l]) == cudaSuccess;
  }
  ok = ok && cudaMallocHost(&h->stage, (size_t)w * hgt) == cudaSuccess;
  if (!ok) { svs_prep_destroy(h); return SVS_ERR_CUDA; }
  *out = h;
  return SVS_OK;
}

void svs_prep_destroy(svs_prep* h) {
  if (!h) return;
  svs::begin_close(h);
  for (int l = 0; l < kMaxLv; ++l) { cudaFree(h->u8[l]); for (int k = 0; k < 3; ++k) cudaFree(h->f32[l][k]); }
  if (h->stage) cudaFreeHost(h->stage);
  delete h;
}

const char* svs_prep_last_error(const svs_prep* h) { return svs::last_error(h); }

int svs_prep_process(svs_prep* h, const unsigned char* img, int pitch) {
  if (!h || !img || pitch < h->w[0]) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  SVS_CK(h, cudaStreamSynchronize(h->stream));   // staging buffer reuse
  for (int y = 0; y < h->h[0]; ++y) memcpy(h->stage + (size_t)y * h->w[0], img + (size_t)y * pitch, h->w[0]);
  SVS_CK(h, cudaMemcpy2DAsync(h->u8[0], h->pitch8[0], h->stage, h->w[0], h->w[0], h->h[0], cudaMemcpyHostToDevice, h->stream));
  const dim3 blk(32, 8);
  auto grid = [&](int w, int hh) { return dim3((w + 31) / 32, (hh + 7) / 8); };
  k_u8_to_f32<<<grid(h->w[0], h->h[0]), blk, 0, h->stream>>>(h->u8[0], h->pitch8[0], h->f32[0][0], h->stride32[0], h->w[0], h->h[0]);
  for (int l = 0; l < h->nlevels; ++l) {
    if (l > 0) {
      k_pyrdown_u8<<<grid(h->w[l], h->h[l]), blk, 0, h->stream>>>(h->u8[l - 1], h->pitch8[l - 1], h->w[l - 1], h->h[l - 1], h->u8[l], h->pitch8[l]);
      k_pyrdown_f32<<<grid(h->w[l], h->h[l]), blk, 0, h->stream>>>(h->f32[l - 1][0], h->stride32[l - 1], h->w[l - 1], h->h[l - 1],
                                                                      h->f32[l][0], h->stride32[l]);
    }
    k_deriv<<<grid(h->w[l], h->h[l]), blk, 0, h->stream>>>(h->f32[l][0], h->stride32[l], h->w[l], h->h[l], h->f32[l][1], h->f32[l][2]);
  }
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaStreamSynchronize(h->stream));   // consumers run on their own streams
  return SVS_OK;
}

int svs_prep_level(svs_prep* h, int level, int* w, int* hgt, const unsigned char** u8, int* pitch_u8, const float** f32,
                   const float** dx, const float** dy, int* stride_f32) {
  if (!h || level < 0 || level >= h->nlevels) return SVS_ERR_INVALID;
  if (w) *w = h->w[level];
  if (hgt) *hgt = h->h[level];
  if (u8) *u8 = h->u8[level];
  if (pitch_u8) *pitch_u8 = h->pitch8[level];
  if (f32) *f32 = h->f32[level][0];
  if (dx) *dx = h->f32[level][1];
  if (dy) *dy = h->f32[level][2];
  if (stride_f32) *stride_f32 = h->stride32[level];
  return SVS_OK;
}

int svs_prep_get_u8(svs_prep* h, int level, unsigned char* out) {
  if (!h || level < 0 || level >= h->nlevels || !out) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpy2D(out, h->w[level], h->u8[level], h->pitch8[level], h->w[level], h->h[level], cudaMemcpyDeviceToHost));
  return SVS_OK;
}

int svs_prep_get_f32(svs_prep* h, int level, int which, float* out) {
  if (!h || level < 0 || level >= h->nlevels || which < 0 || which > 2 || !out) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpy2D(out, sizeof(float) * h->w[level], h->f32[level][which], sizeof(float) * h->stride32[level],
                         sizeof(float) * h->w[level], h->h[level], cudaMemcpyDeviceToHost));
  return SVS_OK;
}

}  // extern "C"
