// dtc.cu -- the dense tracker the reference builds WITHOUT SCAVISLAM_CUDA_SUPPORT (SURVEY.md 8 row a18):
// DenseTracker::denseTrackingCpu / computeDensePointCloudCpu (scavislam/dense_tracking.cpp:222-423),
// on sm_90a.  Semantics that differ from the CUDA build of the reference (dt.cu follows that one):
// every 4th pixel in u and v (EVERY_NTH_PIXEL, dense_tracking.h:82), the previous intensity comes from
// the uint8 pyramid, residual clamped to +-0.1, exact software bilinear taps (interpolateMat_32f,
// maths_utils.cpp:46-65), FP64 point transform and Jacobian, border test isInFrame(uv, 2), the
// disparity is scaled by 2^-level, and H is NOT damped (mu is updated but never applied, :332).
//
// The grid is (w/4) x (h/4) points per level -- 19 200 at 640x480 -- so one CTA runs the whole
// coarse-to-fine Levenberg loop of a level on the device: a sweep at a trial pose yields chi2, H and
// J^T r at once (an accepted step costs one sweep); fixed-order FP64 block reduction (the reference sums
// sequentially in FP32: documented deviation D-DT4); 6x6 LDL^T and exp(x) T by thread 0.
// Per-pixel float arithmetic is the reference's, operation by operation (compiled with -fmad=false).
#include <cmath>
#include <cstring>
#include <string>

#include <cuda_runtime.h>

#include "../../include/svs_b200.h"
#include "handle.cuh"
#include "se3_dev.cuh"
#include "svs_nvtx.hpp"

namespace {

constexpr int kNth = 4;
constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kAcc = 28;   // 21 H (upper triangle), 6 J^T r, chi2
constexpr int kMaxLv = 8;

struct DtcLevel {
  int w, h, stride, pitch_u8;
  double f, px, py;
  const unsigned char* prev_u8;
  const float* cur;
  const float* dx;
  const float* dy;
  const float4* cloud;   // (h/4) x (w/4)
};

struct DtcCtl {
  double T[7];
  double chi2[kMaxLv];
  int passes[kMaxLv];
};

// interpolateMat_32f (maths_utils.cpp:46-65)
__device__ __forceinline__ float interp32f(const float* __restrict__ img, int stride, float u, float v) {
  const float x = floorf(u), y = floorf(v);
  const float sx = u - x, sy = v - y;
  const float wx0 = 1 - sx, wx1 = sx, wy0 = 1 - sy, wy1 = sy;
  const float* p = img + (size_t)(int)y * stride + (int)x;
  const float v00 = __ldg(p), v01 = __ldg(p + stride), v10 = __ldg(p + 1), v11 = __ldg(p + stride + 1);
  return (wx0 * wy0) * v00 + (wx0 * wy1) * v01 + (wx1 * wy0) * v10 + (wx1 * wy1) * v11;
}

__device__ void sweep(const DtcLevel& L, const double R[9], const double t[3], double acc[kAcc]) {
#pragma unroll
  for (int k = 0; k < kAcc; ++k) acc[k] = 0.;
  const int gw = L.w / kNth, n = gw * (L.h / kNth);
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const float4 c4 = __ldg(L.cloud + i);
    if (!(c4.w > 0)) continue;
    const int v = i / gw, u = i - v * gw;
    const double X = c4.x, Y = c4.y, Z = c4.z;
    const double x = R[0] * X + R[1] * Y + R[2] * Z + t[0];
    const double y = R[3] * X + R[4] * Y + R[5] * Z + t[1];
    const double z = R[6] * X + R[7] * Y + R[8] * Z + t[2];
    const float uc = (float)(L.f * (x / z) + L.px), vc = (float)(L.f * (y / z) + L.py);
    const int ui = (int)uc, vi = (int)vc;
    if (!(ui >= 2 && ui < L.w - 2 && vi >= 2 && vi < L.h - 2)) continue;
    const float ip = (float)((1. / 255.) * (double)__ldg(L.prev_u8 + (size_t)(v * kNth) * L.pitch_u8 + u * kNth));
    const float ic = interp32f(L.cur, L.stride, uc, vc);
    float res = ip - ic;
    if (res > 0.1) res = 0.1f;
    if (res < -0.1) res = -0.1f;
    acc[27] += (double)(res * res);
    const float dx = (float)(0.5 * (double)interp32f(L.dx, L.stride, uc, vc));
    const float dy = (float)(0.5 * (double)interp32f(L.dy, L.stride, uc, vc));
    // frame_jac_xyz2uv (transformations.h:116-140)
    const double z2 = z * z, f = L.f;
    const double r0[6] = {-1. / z * f, 0, x / z2 * f, x * y / z2 * f, -(1 + (x * x / z2)) * f, y / z * f};
    const double r1[6] = {0, -1. / z * f, y / z2 * f, (1 + y * y / z2) * f, -x * y / z2 * f, -x / z * f};
    double J[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) J[k] = (double)dx * r0[k] + (double)dy * r1[k];
    int q = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
#pragma unroll
      for (int c = r; c < 6; ++c) acc[q++] += J[r] * J[c];
      acc[21 + r] += J[r] * (double)res;
    }
  }
}

struct Shared {
  double part[kWarps][kAcc];
  double sum[kAcc];
  double R[9], t[3];
  int go;
};

__device__ void reduce(Shared& sh, double acc[kAcc]) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kAcc; ++k) {
    double s = acc[k];
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) sh.part[w][k] = s;
  }
  __syncthreads();
  if (threadIdx.x < kAcc) {
    double s = 0;
    for (int q = 0; q < kWarps; ++q) s += sh.part[q][threadIdx.x];
    sh.sum[threadIdx.x] = s;
  }
  __syncthreads();
}

// H x = -Jres (Eigen ldlt() in the reference; a zero pivot gives a zero component instead of NaN)
__device__ void solve6(const double* H21, const double* Jr, double x[6]) {
  double A[6][6], Lm[6][6], D[6], y[6];
  int q = 0;
  for (int r = 0; r < 6; ++r)
    for (int c = r; c < 6; ++c) { A[r][c] = A[c][r] = H21[q++]; }
  for (int j = 0; j < 6; ++j) {
    double d = A[j][j];
    for (int k = 0; k < j; ++k) d -= Lm[j][k] * Lm[j][k] * D[k];
    D[j] = d;
    for (int i = j + 1; i < 6; ++i) {
      double s = A[i][j];
      for (int k = 0; k < j; ++k) s -= Lm[i][k] * Lm[j][k] * D[k];
      Lm[i][j] = d != 0. ? s / d : 0.;
    }
  }
  for (int i = 0; i < 6; ++i) {
    double s = -Jr[i];
    for (int k = 0; k < i; ++k) s -= Lm[i][k] * y[k];
    y[i] = s;
  }
  for (int i = 5; i >= 0; --i) {
    double s = D[i] != 0. ? y[i] / D[i] : 0.;
    for (int k = i + 1; k < 6; ++k) s -= Lm[k][i] * x[k];
    x[i] = s;
  }
}

__device__ void propose(Shared& sh, const double* H, const double* Jr, const double T[7], double Tn[7], double x[6]) {
  double dT[7];
  solve6(H, Jr, x);
  svs::se3_exp(x, dT);
  svs::se3_mul(dT, T, Tn);
  svs::quat_to_R(Tn, sh.R);
  sh.t[0] = Tn[4]; sh.t[1] = Tn[5]; sh.t[2] = Tn[6];
}

// denseTrackingCpu for one level (dense_tracking.cpp:225-391)
__global__ void __launch_bounds__(kThreads) k_dtc_level(DtcLevel L, DtcCtl* ctl, int level) {
  __shared__ Shared sh;
  double T[7], Tn[7], H[21], Jr[6], x[6], chi2 = 0;
  int iter = 0, passes = 1;
  if (threadIdx.x == 0) {
    for (int k = 0; k < 7; ++k) T[k] = ctl->T[k];
    svs::quat_to_R(T, sh.R);
    sh.t[0] = T[4]; sh.t[1] = T[5]; sh.t[2] = T[6];
  }
  __syncthreads();
  double acc[kAcc];
  {
    double R[9], t[3];
    for (int k = 0; k < 9; ++k) R[k] = sh.R[k];
    for (int k = 0; k < 3; ++k) t[k] = sh.t[k];
    sweep(L, R, t, acc);
  }
  reduce(sh, acc);
  if (threadIdx.x == 0) {
    for (int k = 0; k < 21; ++k) H[k] = sh.sum[k];
    for (int k = 0; k < 6; ++k) Jr[k] = sh.sum[21 + k];
    chi2 = sh.sum[27];
    sh.go = 1;
    propose(sh, H, Jr, T, Tn, x);
  }
  __syncthreads();
  while (sh.go) {
    double R[9], t[3];
    for (int k = 0; k < 9; ++k) R[k] = sh.R[k];
    for (int k = 0; k < 3; ++k) t[k] = sh.t[k];
    __syncthreads();
    sweep(L, R, t, acc);
    reduce(sh, acc);
    if (threadIdx.x == 0) {
      ++passes;
      const double rho = chi2 - sh.sum[27];
      bool stop;
      if (rho > 0) {   // :368-376
        for (int k = 0; k < 7; ++k) T[k] = Tn[k];
        chi2 = sh.sum[27];
        for (int k = 0; k < 21; ++k) H[k] = sh.sum[k];
        for (int k = 0; k < 6; ++k) Jr[k] = sh.sum[21 + k];
        double nm = 0;
        for (int k = 0; k < 6; ++k) nm = fmax(nm, fabs(x[k]));
        stop = nm <= 0.0000000001;
        ++iter;
      } else {         // :378-385: the reference repeats the identical trial, rejects it again and stops
        stop = true;
      }
      if (stop || iter >= 15) sh.go = 0;
      else propose(sh, H, Jr, T, Tn, x);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    for (int k = 0; k < 7; ++k) ctl->T[k] = T[k];
    ctl->chi2[level] = chi2; ctl->passes[level] = passes;
  }
}

// computeDensePointCloudCpu for one level (dense_tracking.cpp:393-422); TQ row-major, FP64
struct M4d { double m[16]; };
__global__ void k_dtc_pointcloud(M4d TQ, const float* __restrict__ disp, int disp_stride, int level, int gw, int gh,
                                 float4* __restrict__ cloud) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x, v = blockIdx.y * blockDim.y + threadIdx.y;
  if (u >= gw || v >= gh) return;
  const double inv_factor = 1. / (double)(1 << level);
  const double d = (double)__ldg(disp + (size_t)((v * 4) << level) * disp_stride + ((u * 4) << level)) * inv_factor;
  float4 o;
  if (d <= 0) {
    o = make_float4(0.f, 0.f, 0.f, -1.f);
  } else {
    const double uvd[4] = {(double)(u * kNth), (double)(v * kNth), d, 1.};
    double p[4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
      p[r] = TQ.m[r * 4] * uvd[0] + TQ.m[r * 4 + 1] * uvd[1] + TQ.m[r * 4 + 2] * uvd[2] + TQ.m[r * 4 + 3] * uvd[3];
    o = make_float4((float)(p[0] / p[3]), (float)(p[1] / p[3]), (float)(p[2] / p[3]), 1.f);
  }
  cloud[(size_t)v * gw + u] = o;
}

}  // namespace

struct svs_dtc : svs::Handle {
  int nlevels = 0, w0 = 0, h0 = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int w[kMaxLv] = {}, h[kMaxLv] = {}, stride[kMaxLv] = {}, pitch8[kMaxLv] = {};
  unsigned char* prev8[kMaxLv] = {};
  float* img[kMaxLv][3] = {};   // cur dx dy
  float4* cloud[kMaxLv] = {};
  float* disp = nullptr;
  int disp_stride = 0;
  DtcCtl* d_ctl = nullptr;
  DtcCtl* h_ctl = nullptr;
};

extern "C" {

int svs_dtc_create(int device, int w0, int h0, int nlevels, svs_dtc** out) {
  if (!out || w0 <= 0 || h0 <= 0 || nlevels <= 0 || nlevels > kMaxLv) return SVS_ERR_INVALID;
  *out = nullptr;
  for (int l = 0; l < nlevels; ++l)   // the reference asserts the same (dense_tracking.cpp:42-43)
    if (((w0 >> l) % kNth) || ((h0 >> l) % kNth) || (w0 >> l) < 8 || (h0 >> l) < 8) return SVS_ERR_INVALID;
  svs_dtc* h = new svs_dtc();
  if (int rc = svs::open_handle(h, device)) {
    delete h;
    return rc;
  }
  h->nlevels = nlevels; h->w0 = w0; h->h0 = h0;
  bool ok = cudaEventCreate(&h->ev0) == cudaSuccess && cudaEventCreate(&h->ev1) == cudaSuccess;
  for (int l = 0; ok && l < nlevels; ++l) {
    h->w[l] = w0 >> l; h->h[l] = h0 >> l;
    h->stride[l] = ((h->w[l] + 63) / 64) * 64;
    h->pitch8[l] = ((h->w[l] + 255) / 256) * 256;
    ok = cudaMalloc(&h->prev8[l], (size_t)h->pitch8[l] * h->h[l]) == cudaSuccess &&
         cudaMemset(h->prev8[l], 0, (size_t)h->pitch8[l] * h->h[l]) == cudaSuccess;
    for (int k = 0; ok && k < 3; ++k)
      ok = cudaMalloc(&h->img[l][k], sizeof(float) * (size_t)h->stride[l] * h->h[l]) == cudaSuccess &&
           cudaMemset(h->img[l][k], 0, sizeof(float) * (size_t)h->stride[l] * h->h[l]) == cudaSuccess;
    const size_t npts = (size_t)(h->w[l] / kNth) * (h->h[l] / kNth);
    ok = ok && cudaMalloc(&h->cloud[l], sizeof(float4) * npts) == cudaSuccess &&
         cudaMemset(h->cloud[l], 0, sizeof(float4) * npts) == cudaSuccess;
  }
  h->disp_stride = ((w0 + 63) / 64) * 64;
  ok = ok && cudaMalloc(&h->disp, sizeof(float) * (size_t)h->disp_stride * h0) == cudaSuccess &&
       cudaMemset(h->disp, 0, sizeof(float) * (size_t)h->disp_stride * h0) == cudaSuccess &&
       cudaMalloc(&h->d_ctl, sizeof(DtcCtl)) == cudaSuccess && cudaMallocHost(&h->h_ctl, sizeof(DtcCtl)) == cudaSuccess;
  if (!ok) { svs_dtc_destroy(h); return SVS_ERR_CUDA; }
  *out = h;
  return SVS_OK;
}

void svs_dtc_destroy(svs_dtc* h) {
  if (!h) return;
  svs::begin_close(h);
  for (int l = 0; l < kMaxLv; ++l) {
    cudaFree(h->prev8[l]); cudaFree(h->cloud[l]);
    for (int k = 0; k < 3; ++k) cudaFree(h->img[l][k]);
  }
  cudaFree(h->disp); cudaFree(h->d_ctl);
  if (h->h_ctl) cudaFreeHost(h->h_ctl);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  delete h;
}

const char* svs_dtc_last_error(const svs_dtc* h) { return svs::last_error(h); }

int svs_dtc_set_prev_u8(svs_dtc* h, int level, const unsigned char* img, int pitch, int on_device) {
  if (!h || level < 0 || level >= h->nlevels || !img || pitch < h->w[level]) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpy2DAsync(h->prev8[level], h->pitch8[level], img, pitch, h->w[level], h->h[level],
                              on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, h->stream));
  if (!on_device) SVS_CK(h, cudaStreamSynchronize(h->stream));   // pageable source may be reused by the caller
  return SVS_OK;
}

int svs_dtc_set_cur(svs_dtc* h, int level, const float* cur, const float* dx, const float* dy, int stride_floats, int on_device) {
  if (!h || level < 0 || level >= h->nlevels || stride_floats < h->w[level]) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  const float* src[3] = {cur, dx, dy};
  for (int k = 0; k < 3; ++k)
    if (src[k])
      SVS_CK(h, cudaMemcpy2DAsync(h->img[level][k], sizeof(float) * h->stride[level], src[k], sizeof(float) * stride_floats,
                                  sizeof(float) * h->w[level], h->h[level],
                                  on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, h->stream));
  if (!on_device) SVS_CK(h, cudaStreamSynchronize(h->stream));
  return SVS_OK;
}

int svs_dtc_set_disparity(svs_dtc* h, const float* disp, int stride_floats) {
  if (!h || !disp || stride_floats < h->w0) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpy2DAsync(h->disp, sizeof(float) * h->disp_stride, disp, sizeof(float) * stride_floats, sizeof(float) * h->w0,
                              h->h0, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  return SVS_OK;
}

// the same map already on this device (svs_stereo_disparity): a device-to-device copy; on return the source may change
int svs_dtc_set_disparity_device(svs_dtc* h, const float* d_disp, int stride_floats) {
  if (!h || !d_disp || stride_floats < h->w0) return SVS_ERR_INVALID;
  if (!svs::on_device(h->device, d_disp)) return svs::fail(h, SVS_ERR_INVALID, "svs_dtc_set_disparity_device: not device memory of this handle's device");
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpy2DAsync(h->disp, sizeof(float) * h->disp_stride, d_disp, sizeof(float) * stride_floats, sizeof(float) * h->w0,
                              h->h0, cudaMemcpyDeviceToDevice, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  return SVS_OK;
}

int svs_computeDensePointCloudCpu(svs_dtc* h, const double T[7], const svs_cam* cams) {
  svs::NvtxRange nvtx_("dense point cloud");
  if (!h || !T || !cams) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  // T^-1 (Sophus inverse: conjugate quaternion, -R^T t)
  const double x = -T[0], y = -T[1], z = -T[2], w = T[3];
  const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                       2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                       2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
  double ti[3];
  for (int r = 0; r < 3; ++r) ti[r] = -(R[r * 3] * T[4] + R[r * 3 + 1] * T[5] + R[r * 3 + 2] * T[6]);
  for (int l = 0; l < h->nlevels; ++l) {
    const svs_cam& c = cams[l];
    const double M[16] = {R[0], R[1], R[2], ti[0], R[3], R[4], R[5], ti[1], R[6], R[7], R[8], ti[2], 0, 0, 0, 1};
    const double Q[16] = {1, 0, 0, -c.px, 0, 1, 0, -c.py, 0, 0, 0, c.f, 0, 0, 1. / c.b, 0};   // stereo_camera.cpp:24-34
    M4d TQ;
    for (int r = 0; r < 4; ++r)
      for (int cc = 0; cc < 4; ++cc) {
        double s = 0;
        for (int k = 0; k < 4; ++k) s += M[r * 4 + k] * Q[k * 4 + cc];
        TQ.m[r * 4 + cc] = s;
      }
    const int gw = h->w[l] / kNth, gh = h->h[l] / kNth;
    const dim3 blk(32, 8), grd((gw + 31) / 32, (gh + 7) / 8);
    k_dtc_pointcloud<<<grd, blk, 0, h->stream>>>(TQ, h->disp, h->disp_stride, l, gw, gh, h->cloud[l]);
  }
  SVS_CK(h, cudaGetLastError());
  return SVS_OK;
}

int svs_dtc_get_point_cloud(svs_dtc* h, int level, float* cloud_xyzw) {
  if (!h || level < 0 || level >= h->nlevels || !cloud_xyzw) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  const size_t npts = (size_t)(h->w[level] / kNth) * (h->h[level] / kNth);
  SVS_CK(h, cudaMemcpyAsync(cloud_xyzw, h->cloud[level], sizeof(float4) * npts, cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  return SVS_OK;
}

int svs_dtc_set_point_cloud(svs_dtc* h, int level, const float* cloud_xyzw) {
  if (!h || level < 0 || level >= h->nlevels || !cloud_xyzw) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  const size_t npts = (size_t)(h->w[level] / kNth) * (h->h[level] / kNth);
  SVS_CK(h, cudaMemcpyAsync(h->cloud[level], cloud_xyzw, sizeof(float4) * npts, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  return SVS_OK;
}

int svs_denseTrackingCpu(svs_dtc* h, const svs_cam* cams, double T[7], svs_dt_stats* st) {
  svs::NvtxRange nvtx_("dense tracking");
  if (!h || !cams || !T) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  memcpy(h->h_ctl->T, T, sizeof(double) * 7);
  SVS_CK(h, cudaMemcpyAsync(h->d_ctl, h->h_ctl, sizeof(double) * 7, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaEventRecord(h->ev0, h->stream));
  for (int l = h->nlevels - 1; l >= 0; --l) {
    DtcLevel L;
    L.w = h->w[l]; L.h = h->h[l]; L.stride = h->stride[l]; L.pitch_u8 = h->pitch8[l];
    L.f = cams[l].f; L.px = cams[l].px; L.py = cams[l].py;
    L.prev_u8 = h->prev8[l]; L.cur = h->img[l][0]; L.dx = h->img[l][1]; L.dy = h->img[l][2]; L.cloud = h->cloud[l];
    k_dtc_level<<<1, kThreads, 0, h->stream>>>(L, h->d_ctl, l);
  }
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaEventRecord(h->ev1, h->stream));
  SVS_CK(h, cudaMemcpyAsync(h->h_ctl, h->d_ctl, sizeof(DtcCtl), cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  memcpy(T, h->h_ctl->T, sizeof(double) * 7);
  if (st) {
    memset(st, 0, sizeof *st);
    cudaEventElapsedTime(&st->ms_total, h->ev0, h->ev1);
    for (int l = 0; l < h->nlevels && l < SVS_DT_MAX_LEVELS; ++l) {
      st->chi2[l] = h->h_ctl->chi2[l]; st->passes[l] = h->h_ctl->passes[l]; st->launches += 1;
    }
  }
  return SVS_OK;
}

}  // extern "C"
