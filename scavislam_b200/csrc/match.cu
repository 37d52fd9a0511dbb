// match.cu -- guided patch matcher on sm_90a: GuidedMatcher<StereoCamera>::match
// (scavislam/matcher.cpp:312-398) with computePrediction (:98-142), warpAffinve (:403-458),
// computePatchScores (:77-96), matchCandidates / matchPatchZeroMeanSSD (:42-74, :144-181),
// returnBestMatch (:183-216) and createObervation (matcher-impl.cpp:32-51).
//
// One warp per candidate 3-D point.  The reference's FAST quadtree (quadtree.h) is replaced by
// a bucket grid over the keypoints of each pyramid level; the quadtree only matters through the
// order in which it enumerates candidates (the strict `<` keeps the FIRST best score), which is
// the Z-order of recursive midpoint subdivision with x before y -- reproduced by an explicit
// (score, z-key) minimum, so the result does not depend on enumeration order.
// Integer scores are exact; the double-precision prediction/warp chain is compiled with
// -fmad=false and written operation by operation like the CPU oracle so that the uint8
// truncation of the warped patch is bit-identical.
#include <algorithm>
#include <cstddef>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/svs_b200.h"
#include "handle.cuh"
#include "internal.cuh"
#include "se3_dev.cuh"
#include "svs_nvtx.hpp"

namespace {

constexpr int kMaxLv = SVS_MATCH_MAX_LEVELS;
constexpr int kBucket = 16;
constexpr int kWarps = 4;

struct LvDev {
  int w, h;
  double f, px, py;
  const unsigned char* cur;   // current frame, this level
  int cur_pitch;
  const int* kp_xy;           // [n][2]
  const int* kp_content;      // [n]
  const int* bucket_ptr;      // [(bw*bh)+1]
  const int* bucket_item;     // [n]
  int nkp, bw, bh;
};

struct KfDev {
  double T[7];
  const unsigned char* pyr[kMaxLv];
  int pitch[kMaxLv];
};

struct MatchArgs {
  LvDev lv[kMaxLv];
  int nlevels;
  const KfDev* kf;
  int nkf;
  const float* disp;
  int disp_pitch;
  double T_cur_from_actkey[7];
  double T_actkey_from_w[7];
  int radius, thr_mean, thr_std;
};

__device__ __forceinline__ void se3_act(const double A[7], const double x[3], double y[3]) {
  double R[9];
  svs::quat_to_R(A, R);
  svs::mat3_vec(R, x, y);
  y[0] += A[4]; y[1] += A[5]; y[2] += A[6];
}

__device__ __forceinline__ void cam_map(const LvDev& L, const double xyz[3], double uv[2]) {
  uv[0] = L.f * (xyz[0] / xyz[2]) + L.px;
  uv[1] = L.f * (xyz[1] / xyz[2]) + L.py;
}

__device__ __forceinline__ bool in_frame(const LvDev& L, int u, int v, int border) {
  return u >= border && u < L.w - border && v >= border && v < L.h - border;
}

// position of (x, y) along the quadtree's depth-first enumeration (quadtree.h:511-545, 679-710)
__device__ __forceinline__ unsigned zkey(int x, int y, int w, int h) {
  const unsigned tx = (unsigned)(((long long)x << 12) / w), ty = (unsigned)(((long long)y << 12) / h);
  unsigned k = 0;
#pragma unroll
  for (int b = 0; b < 12; ++b) k |= (((tx >> b) & 1u) << (2 * b + 1)) | (((ty >> b) & 1u) << (2 * b));
  return k;
}

__global__ void __launch_bounds__(kWarps * 32)
k_match(MatchArgs a, const svs_match_point* __restrict__ pts, int n, svs_match_result* __restrict__ res) {
  __shared__ unsigned char s_patch[kWarps][104];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * kWarps + warp;
  if (i >= n) return;
  const svs_match_point ap = pts[i];
  svs_match_result r;
  memset(&r, 0, sizeof r);
  r.index = -1;
  bool alive = ap.keyframe >= 0 && ap.keyframe < a.nkf && ap.anchor_level >= 0 && ap.anchor_level < a.nlevels;
  const int lv = alive ? ap.anchor_level : 0;
  const LvDev& L = a.lv[lv];
  double T_cur_from_anchor[7];
  int ui = 0, vi = 0;
  if (alive) {
    const KfDev& kf = a.kf[ap.keyframe];
    // T_cur_from_w = T_cur_from_actkey * T_actkey_from_w (matcher.cpp:327-331)
    double Tai[7], xyz_cur[3], uv_pyr[2], T_cur_from_w[7];
    svs::se3_mul(a.T_cur_from_actkey, a.T_actkey_from_w, T_cur_from_w);
    svs::se3_inv(kf.T, Tai);
    svs::se3_mul(T_cur_from_w, Tai, T_cur_from_anchor);
    se3_act(T_cur_from_anchor, ap.xyz_anchor, xyz_cur);
    cam_map(L, xyz_cur, uv_pyr);
    if (!in_frame(L, (int)ap.anchor_obs_pyr[0], (int)ap.anchor_obs_pyr[1], 4)) alive = false;
    const double depth_cur = 1. / xyz_cur[2], depth_anchor = 1. / ap.xyz_anchor[2];
    if (depth_cur > depth_anchor * 3 || depth_anchor > depth_cur * 3) alive = false;
    ui = (int)uv_pyr[0]; vi = (int)uv_pyr[1];
  }
  if (!alive) {
    if (lane == 0) res[i] = r;
    return;
  }
  r.predicted = 1;
  // ---- warpAffinve: 10x10 patch of the anchor keyframe, lanes take pixels lane, lane+32, ...
  {
    const KfDev& kf = a.kf[ap.keyframe];
    const unsigned char* frame = kf.pyr[lv];
    const int pitch = kf.pitch[lv];
    double f0[2], fu[2], fv[2];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double ox = k == 1 ? 1. : 0., oy = k == 2 ? 1. : 0.;
      const double ux = (ap.anchor_obs_pyr[0] + ox - L.px) / L.f, uy = (ap.anchor_obs_pyr[1] + oy - L.py) / L.f;
      const double depth = ap.xyz_anchor[2];
      const double p[3] = {depth * ux, depth * uy, depth * 1.};
      double q[3];
      se3_act(T_cur_from_anchor, p, q);
      cam_map(L, q, k == 0 ? f0 : (k == 1 ? fu : fv));
    }
    const double a00 = fu[0] - f0[0], a01 = fu[1] - f0[1], a10 = fv[0] - f0[0], a11 = fv[1] - f0[1];
    const double det = a00 * a11 - a01 * a10;
    const double idet = 1. / det;
    const double i00 = a11 * idet, i01 = -a01 * idet, i10 = -a10 * idet, i11 = a00 * idet;
    for (int idx = lane; idx < 100; idx += 32) {
      const int iy = idx / 10, ix = idx - iy * 10;
      const double dx = ix - 5, dy = iy - 5;
      const double rx = (i00 * dx + i01 * dy) + ap.anchor_obs_pyr[0];
      const double ry = (i10 * dx + i11 * dy) + ap.anchor_obs_pyr[1];
      const double x = floor(rx), y = floor(ry);
      unsigned char val;
      if (x < 0 || y < 0 || x + 1 >= L.w || y + 1 >= L.h) {
        val = 0;
      } else {
        const double sx = rx - x, sy = ry - y;
        const double wx0 = 1 - sx, wx1 = sx, wy0 = 1 - sy, wy1 = sy;
        const int xi = (int)x, yi = (int)y;
        const double v00 = frame[yi * pitch + xi], v01 = frame[(yi + 1) * pitch + xi];
        const double v10 = frame[yi * pitch + xi + 1], v11 = frame[(yi + 1) * pitch + xi + 1];
        const double s = (wx0 * wy0) * v00 + (wx0 * wy1) * v01 + (wx1 * wy0) * v10 + (wx1 * wy1) * v11;
        val = (unsigned char)(s < 255. ? s : 255.);
      }
      s_patch[warp][iy * 10 + ix] = val;
    }
  }
  __syncwarp();
  // this lane's two pixels of the inner 8x8 key patch: (row, col) and (row + 4, col)
  const int prow = lane >> 3, pcol = lane & 7;
  const int k0 = s_patch[warp][(prow + 1) * 10 + pcol + 1], k1 = s_patch[warp][(prow + 5) * 10 + pcol + 1];
  int sumA = k0 + k1, sumAA = k0 * k0 + k1 * k1;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sumA += __shfl_xor_sync(0xffffffffu, sumA, o);
    sumAA += __shfl_xor_sync(0xffffffffu, sumAA, o);
  }
  if (sumA * sumA - sumAA < (int)(a.thr_std * a.thr_std * 64)) {   // matcher.cpp:384-386 (literal, SURVEY B8)
    if (lane == 0) res[i] = r;
    return;
  }
  r.textured = 1;
  // ---- matchCandidates over the FAST corners in the (2r+1)^2 window
  int min_dist = a.thr_mean * a.thr_mean * 64;
  int best_idx = -1, best_u = 0, best_v = 0, ncand = 0;
  unsigned best_z = 0xffffffffu;
  const int x_lo = ui - a.radius, x_hi = ui + a.radius, y_lo = vi - a.radius, y_hi = vi + a.radius;
  const int bx0 = max(x_lo, 0) / kBucket, bx1 = min(x_hi, L.w - 1) / kBucket;
  const int by0 = max(y_lo, 0) / kBucket, by1 = min(y_hi, L.h - 1) / kBucket;
  if (x_hi >= 0 && y_hi >= 0 && x_lo < L.w && y_lo < L.h) {
    for (int by = by0; by <= by1; ++by)
      for (int bx = bx0; bx <= bx1; ++bx) {
        const int b = by * L.bw + bx;
        const int e0 = L.bucket_ptr[b], e1 = L.bucket_ptr[b + 1];
        for (int e = e0; e < e1; ++e) {
          const int kp = L.bucket_item[e];
          const int cu = L.kp_xy[2 * kp], cv = L.kp_xy[2 * kp + 1];
          if (cu < x_lo || cu > x_hi || cv < y_lo || cv > y_hi) continue;
          ++ncand;
          if (!in_frame(L, cu, cv, 6)) continue;
          const unsigned char* cur = L.cur + (size_t)(cv - 4) * L.cur_pitch + (cu - 4);
          const int b0 = cur[prow * L.cur_pitch + pcol], b1 = cur[(prow + 4) * L.cur_pitch + pcol];
          int sumB = b0 + b1, sumBB = b0 * b0 + b1 * b1, sumAB = b0 * k0 + b1 * k1;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            sumB += __shfl_xor_sync(0xffffffffu, sumB, o);
            sumBB += __shfl_xor_sync(0xffffffffu, sumBB, o);
            sumAB += __shfl_xor_sync(0xffffffffu, sumAB, o);
          }
          // matcher.cpp:73, literal formula with truncating int division (SURVEY B7)
          const int z = sumAA - 2 * sumAB - sumBB - (sumA * sumA - 2 * sumA * sumB - sumB * sumB) / 64;
          const unsigned zk = zkey(cu, cv, L.w, L.h);
          // first strictly-better candidate in quadtree order == minimum of (score, z-key) below the threshold
          if (z < min_dist || (best_idx >= 0 && z == min_dist && zk < best_z)) {
            min_dist = z; best_idx = L.kp_content[kp]; best_u = cu; best_v = cv; best_z = zk;
          }
        }
      }
  }
  r.n_candidates = ncand;
  if (best_idx >= 0) {
    r.index = best_idx; r.min_dist = min_dist; r.uv_pyr[0] = best_u; r.uv_pyr[1] = best_v;
    const double inv_factor = 1. / (double)(1 << lv);
    const double dd = (double)a.disp[(size_t)(best_v << lv) * a.disp_pitch + (best_u << lv)] * inv_factor;
    if (dd > 0) {
      const double s = (double)(1 << lv);
      r.obs[0] = (double)(float)best_u * s; r.obs[1] = (double)(float)best_v * s;
      r.obs[2] = ((double)(float)best_u - dd) * s;
      double Tak[7], Taki[7], T_w_from_actkey[7];
      svs::se3_inv(a.T_actkey_from_w, T_w_from_actkey);
      svs::se3_mul(a.kf[ap.keyframe].T, T_w_from_actkey, Tak);
      svs::se3_inv(Tak, Taki);
      se3_act(Taki, ap.xyz_anchor, r.xyz_actkey);
      r.matched = 1;
    }
  }
  if (lane == 0) res[i] = r;
}

__global__ void k_bucket_count(const int* __restrict__ xy, int n, int bw, int* __restrict__ cnt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicAdd(&cnt[(xy[2 * i + 1] / kBucket) * bw + xy[2 * i] / kBucket], 1);
}
__global__ void k_bucket_scan(int* __restrict__ cnt, int nb, int* __restrict__ ptr, int* __restrict__ cursor) {
  // single thread: the grid has a few thousand buckets at most
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    int s = 0;
    for (int b = 0; b < nb; ++b) { ptr[b] = s; cursor[b] = s; s += cnt[b]; }
    ptr[nb] = s;
  }
}
__global__ void k_bucket_fill(const int* __restrict__ xy, int n, int bw, int* __restrict__ cursor, int* __restrict__ item) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) item[atomicAdd(&cursor[(xy[2 * i + 1] / kBucket) * bw + xy[2 * i] / kBucket], 1)] = i;
}

}  // namespace

struct svs_matcher : svs::Handle {
  int nlevels = 0, max_kf = 0, max_pts = 0, max_kp = 0;
  svs_match_level lv[kMaxLv];
  int pitch[kMaxLv] = {};
  unsigned char* d_cur[kMaxLv] = {};
  std::vector<unsigned char*> d_kfimg;   // [max_kf * nlevels]
  KfDev* d_kf = nullptr;
  std::vector<KfDev> h_kf;
  float* d_disp = nullptr;
  int disp_pitch = 0;
  int* d_kp_xy[kMaxLv] = {};
  int* d_kp_content[kMaxLv] = {};
  int* d_bucket_ptr[kMaxLv] = {};
  int* d_bucket_item[kMaxLv] = {};
  int* d_bucket_tmp[kMaxLv] = {};   // counts + cursor
  int nkp[kMaxLv] = {}, bw[kMaxLv] = {}, bh[kMaxLv] = {};
  svs_match_point* d_pts = nullptr;
  svs_match_result* d_res = nullptr;
  int last_n = 0;   // candidate points of the last svs_match (results stay in d_res)
  int last_pts_own = 0;                 // the last match read its candidates from d_pts
  unsigned long long match_serial = 0;  // counts every match on the handle
  svs::FrontState* front = nullptr;     // frontend_points.cu's state, allocated on first use
};

namespace svs {
void matcher_device_results(svs_matcher* m, const svs_match_result** d_res, int* n, int* device) {
  *d_res = m->d_res; *n = m->last_n; *device = m->device;
}
void matcher_core(svs_matcher* m, MatcherCore* c) {
  c->device = m->device; c->nlevels = m->nlevels; c->max_pts = m->max_pts; c->max_kp = m->max_kp;
  for (int l = 0; l < kMaxLv; ++l) {
    c->lv[l] = l < m->nlevels ? m->lv[l] : svs_match_level{};
    c->d_kp_xy[l] = m->d_kp_xy[l]; c->nkp[l] = m->nkp[l];
  }
  c->stream = m->stream; c->d_pts = m->d_pts; c->d_res = m->d_res;
  c->d_disp = m->d_disp; c->disp_pitch = m->disp_pitch;
  c->last_n = m->last_n; c->last_pts_own = m->last_pts_own; c->match_serial = m->match_serial;
  c->front = &m->front;
  c->base = m;
}
void matcher_view(svs_matcher* m, MatcherView* v) {
  v->device = m->device; v->nlevels = m->nlevels; v->max_kf = m->max_kf; v->max_pts = m->max_pts;
  for (int l = 0; l < kMaxLv; ++l) v->lv[l] = l < m->nlevels ? m->lv[l] : svs_match_level{};
  v->slot_T = reinterpret_cast<double*>(reinterpret_cast<char*>(m->d_kf) + offsetof(KfDev, T));
  v->slot_stride = sizeof(KfDev);
}
}  // namespace svs

// k_match on n candidate points at d_pts (device memory of the handle's device); the results stay in h->d_res
static int match_launch(svs_matcher* h, const double T_cur_from_actkey[7], const double T_actkey_from_w[7],
                        const svs_match_point* d_pts, int n, int search_radius, int thr_mean, int thr_std) {
  MatchArgs a;
  memset(&a, 0, sizeof a);
  a.nlevels = h->nlevels;
  for (int l = 0; l < h->nlevels; ++l) {
    LvDev& L = a.lv[l];
    L.w = h->lv[l].w; L.h = h->lv[l].h; L.f = h->lv[l].f; L.px = h->lv[l].px; L.py = h->lv[l].py;
    L.cur = h->d_cur[l]; L.cur_pitch = h->pitch[l];
    L.kp_xy = h->d_kp_xy[l]; L.kp_content = h->d_kp_content[l];
    L.bucket_ptr = h->d_bucket_ptr[l]; L.bucket_item = h->d_bucket_item[l];
    L.nkp = h->nkp[l]; L.bw = h->bw[l]; L.bh = h->bh[l];
  }
  a.kf = h->d_kf; a.nkf = h->max_kf;
  a.disp = h->d_disp; a.disp_pitch = h->disp_pitch;
  a.radius = search_radius; a.thr_mean = thr_mean; a.thr_std = thr_std;
  memcpy(a.T_cur_from_actkey, T_cur_from_actkey, sizeof(double) * 7);
  memcpy(a.T_actkey_from_w, T_actkey_from_w, sizeof(double) * 7);
  k_match<<<(n + kWarps - 1) / kWarps, kWarps * 32, 0, h->stream>>>(a, d_pts, n, h->d_res);
  SVS_CK(h, cudaGetLastError());
  return SVS_OK;
}

int svs::match_device(svs_matcher* h, const double T_cur_from_actkey[7], const double T_actkey_from_w[7],
                      const svs_match_point* d_pts, int n, int search_radius, int thr_mean, int thr_std) {
  svs::NvtxRange nvtx_("match");
  h->last_n = 0;
  h->last_pts_own = 0;
  ++h->match_serial;
  if (n < 0 || n > h->max_pts || search_radius < 0) { h->err = "match_device: bad point count or radius"; return SVS_ERR_INVALID; }
  if (n == 0) return SVS_OK;
  cudaSetDevice(h->device);
  const int rc = match_launch(h, T_cur_from_actkey, T_actkey_from_w, d_pts, n, search_radius, thr_mean, thr_std);
  if (rc != SVS_OK) return rc;
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  h->last_n = n;
  return SVS_OK;
}

int svs::match_enqueue_own(svs_matcher* h, const double T_cur_from_actkey[7], const double T_actkey_from_w[7], int n,
                           int search_radius, int thr_mean, int thr_std) {
  h->last_n = 0;
  h->last_pts_own = 1;
  ++h->match_serial;
  if (n == 0) return SVS_OK;
  const int rc = match_launch(h, T_cur_from_actkey, T_actkey_from_w, h->d_pts, n, search_radius, thr_mean, thr_std);
  if (rc != SVS_OK) return rc;
  h->last_n = n;
  return SVS_OK;
}

extern "C" {

int svs_matcher_create(int device, int nlevels, const svs_match_level* levels, int max_keyframes, int max_points,
                     int max_keypoints, svs_matcher ** out) {
  if (!out || !levels || nlevels <= 0 || nlevels > kMaxLv || max_keyframes <= 0 || max_points <= 0 || max_keypoints <= 0)
    return SVS_ERR_INVALID;
  *out = nullptr;
  svs_matcher* h = new svs_matcher();
  if (int rc = svs::open_handle(h, device)) {
    delete h;
    return rc;
  }
  h->nlevels = nlevels; h->max_kf = max_keyframes; h->max_pts = max_points; h->max_kp = max_keypoints;
  bool ok = true;
  h->d_kfimg.assign((size_t)max_keyframes * nlevels, nullptr);
  h->h_kf.assign(max_keyframes, KfDev{});
  for (int l = 0; ok && l < nlevels; ++l) {
    h->lv[l] = levels[l];
    if (levels[l].w <= 0 || levels[l].h <= 0) { ok = false; break; }
    h->pitch[l] = ((levels[l].w + 127) / 128) * 128;
    h->bw[l] = levels[l].w / kBucket + 1; h->bh[l] = levels[l].h / kBucket + 1;
    const size_t img = (size_t)h->pitch[l] * levels[l].h;
    ok = ok && cudaMalloc(&h->d_cur[l], img) == cudaSuccess;
    for (int k = 0; ok && k < max_keyframes; ++k) ok = cudaMalloc(&h->d_kfimg[(size_t)k * nlevels + l], img) == cudaSuccess;
    const int nb = h->bw[l] * h->bh[l];
    ok = ok && cudaMalloc(&h->d_kp_xy[l], sizeof(int) * 2 * (size_t)max_keypoints) == cudaSuccess &&
         cudaMalloc(&h->d_kp_content[l], sizeof(int) * (size_t)max_keypoints) == cudaSuccess &&
         cudaMalloc(&h->d_bucket_ptr[l], sizeof(int) * (nb + 1)) == cudaSuccess &&
         cudaMalloc(&h->d_bucket_item[l], sizeof(int) * (size_t)max_keypoints) == cudaSuccess &&
         cudaMalloc(&h->d_bucket_tmp[l], sizeof(int) * 2 * nb) == cudaSuccess &&
         cudaMemset(h->d_bucket_ptr[l], 0, sizeof(int) * (nb + 1)) == cudaSuccess;
  }
  if (ok) {
    h->disp_pitch = ((levels[0].w + 63) / 64) * 64;
    ok = cudaMalloc(&h->d_disp, sizeof(float) * (size_t)h->disp_pitch * levels[0].h) == cudaSuccess &&
         cudaMemset(h->d_disp, 0, sizeof(float) * (size_t)h->disp_pitch * levels[0].h) == cudaSuccess &&
         cudaMalloc(&h->d_kf, sizeof(KfDev) * max_keyframes) == cudaSuccess &&
         cudaMalloc(&h->d_pts, sizeof(svs_match_point) * (size_t)max_points) == cudaSuccess &&
         cudaMalloc(&h->d_res, sizeof(svs_match_result) * (size_t)max_points) == cudaSuccess;
  }
  if (!ok) {
    svs_matcher_destroy(h);
    return SVS_ERR_CUDA;
  }
  for (int k = 0; k < max_keyframes; ++k)
    for (int l = 0; l < nlevels; ++l) { h->h_kf[k].pyr[l] = h->d_kfimg[(size_t)k * nlevels + l]; h->h_kf[k].pitch[l] = h->pitch[l]; }
  *out = h;
  return SVS_OK;
}

void svs_matcher_destroy(svs_matcher * h) {
  if (!h) return;
  svs::begin_close(h);
  for (int l = 0; l < kMaxLv; ++l) {
    cudaFree(h->d_cur[l]); cudaFree(h->d_kp_xy[l]); cudaFree(h->d_kp_content[l]);
    cudaFree(h->d_bucket_ptr[l]); cudaFree(h->d_bucket_item[l]); cudaFree(h->d_bucket_tmp[l]);
  }
  for (unsigned char* p : h->d_kfimg) cudaFree(p);
  cudaFree(h->d_kf); cudaFree(h->d_disp); cudaFree(h->d_pts); cudaFree(h->d_res);
  svs::front_state_free(h->front);
  delete h;
}

const char* svs_matcher_last_error(const svs_matcher * h) { return svs::last_error(h); }

int svs_matcher_set_keyframe(svs_matcher * h, int slot, const double T_me_from_w[7], const unsigned char* const* pyr,
                           const int* pitch) {
  if (!h || slot < 0 || slot >= h->max_kf || !T_me_from_w || !pyr || !pitch) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  memcpy(h->h_kf[slot].T, T_me_from_w, sizeof(double) * 7);
  for (int l = 0; l < h->nlevels; ++l)
    SVS_CK(h, cudaMemcpy2DAsync(h->d_kfimg[(size_t)slot * h->nlevels + l], h->pitch[l], pyr[l], pitch[l], h->lv[l].w, h->lv[l].h,
                                cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaMemcpyAsync(h->d_kf + slot, &h->h_kf[slot], sizeof(KfDev), cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  return SVS_OK;
}

int svs_matcher_set_current(svs_matcher * h, const unsigned char* const* pyr, const int* pitch, const float* disp,
                          int disp_pitch_floats) {
  if (!h || (pyr && !pitch) || (!pyr && !disp)) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  for (int l = 0; pyr && l < h->nlevels; ++l)
    SVS_CK(h, cudaMemcpy2DAsync(h->d_cur[l], h->pitch[l], pyr[l], pitch[l], h->lv[l].w, h->lv[l].h, cudaMemcpyHostToDevice, h->stream));
  if (disp)
    SVS_CK(h, cudaMemcpy2DAsync(h->d_disp, sizeof(float) * h->disp_pitch, disp, sizeof(float) * disp_pitch_floats,
                                sizeof(float) * h->lv[0].w, h->lv[0].h, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  return SVS_OK;
}

// cur_frame.disp already on this device (svs_stereo_disparity): a device-to-device copy; on return the source may change
int svs_matcher_set_disparity_device(svs_matcher * h, const float* d_disp, int pitch_floats) {
  if (!h || !d_disp || pitch_floats < h->lv[0].w) return SVS_ERR_INVALID;
  if (!svs::on_device(h->device, d_disp)) return svs::fail(h, SVS_ERR_INVALID, "svs_matcher_set_disparity_device: not device memory of this handle's device");
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpy2DAsync(h->d_disp, sizeof(float) * h->disp_pitch, d_disp, sizeof(float) * pitch_floats,
                              sizeof(float) * h->lv[0].w, h->lv[0].h, cudaMemcpyDeviceToDevice, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  return SVS_OK;
}

// Same as set_keyframe / set_current, but the pyramid already lives on this device (svs_prep_level):
// a device-to-device copy into the handle's own buffers, so a keyframe outlives the preprocessor's frame.
int svs_matcher_set_pyramid_device(svs_matcher * h, int which, const double T_me_from_w[7], const unsigned char* const* d_pyr,
                                   const int* pitch) {
  if (!h || which < -1 || which >= h->max_kf || !d_pyr || !pitch || (which >= 0 && !T_me_from_w)) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  for (int l = 0; l < h->nlevels; ++l) {
    unsigned char* dst = which < 0 ? h->d_cur[l] : h->d_kfimg[(size_t)which * h->nlevels + l];
    SVS_CK(h, cudaMemcpy2DAsync(dst, h->pitch[l], d_pyr[l], pitch[l], h->lv[l].w, h->lv[l].h, cudaMemcpyDeviceToDevice, h->stream));
  }
  if (which >= 0) {
    memcpy(h->h_kf[which].T, T_me_from_w, sizeof(double) * 7);
    SVS_CK(h, cudaMemcpyAsync(h->d_kf + which, &h->h_kf[which], sizeof(KfDev), cudaMemcpyHostToDevice, h->stream));
  }
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  return SVS_OK;
}

int svs_matcher_set_features(svs_matcher * h, int level, const int* xy, const int* content, int n) {
  if (!h || level < 0 || level >= h->nlevels || n < 0 || n > h->max_kp || (n && (!xy || !content))) return SVS_ERR_INVALID;
  for (int i = 0; i < n; ++i)
    if (xy[2 * i] < 0 || xy[2 * i] >= h->lv[level].w || xy[2 * i + 1] < 0 || xy[2 * i + 1] >= h->lv[level].h) {
      h->err = "keypoint outside the level image";
      return SVS_ERR_INVALID;
    }
  cudaSetDevice(h->device);
  const int nb = h->bw[level] * h->bh[level];
  h->nkp[level] = n;
  SVS_CK(h, cudaMemsetAsync(h->d_bucket_tmp[level], 0, sizeof(int) * 2 * nb, h->stream));
  if (n) {
    SVS_CK(h, cudaMemcpyAsync(h->d_kp_xy[level], xy, sizeof(int) * 2 * (size_t)n, cudaMemcpyHostToDevice, h->stream));
    SVS_CK(h, cudaMemcpyAsync(h->d_kp_content[level], content, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, h->stream));
    k_bucket_count<<<(n + 255) / 256, 256, 0, h->stream>>>(h->d_kp_xy[level], n, h->bw[level], h->d_bucket_tmp[level]);
  }
  k_bucket_scan<<<1, 32, 0, h->stream>>>(h->d_bucket_tmp[level], nb, h->d_bucket_ptr[level], h->d_bucket_tmp[level] + nb);
  if (n)
    k_bucket_fill<<<(n + 255) / 256, 256, 0, h->stream>>>(h->d_kp_xy[level], n, h->bw[level], h->d_bucket_tmp[level] + nb,
                                                          h->d_bucket_item[level]);
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaStreamSynchronize(h->stream));   // host arrays may go away
  return SVS_OK;
}

// FAST corners handed over on the device (FastGrid::detect fills the quadtree the matcher queries,
// fast_grid.cpp:75-80: content = index of the corner inside its cell): no trip through host memory.
__global__ void k_kp_from_fast(const int* __restrict__ xy, const int* __restrict__ cell_off, int ncells, int n,
                               int* __restrict__ kp_xy, int* __restrict__ kp_content) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int c = 0;
  while (c + 1 < ncells && cell_off[c + 1] <= i) ++c;
  kp_xy[2 * i] = xy[2 * i]; kp_xy[2 * i + 1] = xy[2 * i + 1];
  kp_content[i] = i - cell_off[c];
}

int svs_matcher_set_features_from_fast(svs_matcher * h, int level, svs_fast* fast) {
  if (!h || !fast || level < 0 || level >= h->nlevels) return SVS_ERR_INVALID;
  const int* d_xy; const int* d_off; int ncells, n, dev;
  svs::fast_device_results(fast, &d_xy, &d_off, &ncells, &n, &dev);
  if (dev != h->device) { h->err = "FAST handle lives on another device"; return SVS_ERR_INVALID; }
  if (n < 0 || n > h->max_kp) { h->err = "more keypoints than the matcher was created for"; return SVS_ERR_INVALID; }
  cudaSetDevice(h->device);
  const int nb = h->bw[level] * h->bh[level];
  h->nkp[level] = n;
  SVS_CK(h, cudaMemsetAsync(h->d_bucket_tmp[level], 0, sizeof(int) * 2 * nb, h->stream));
  if (n) {
    // the detect call synchronised the FAST handle's stream before it returned: its results are complete
    k_kp_from_fast<<<(n + 255) / 256, 256, 0, h->stream>>>(d_xy, d_off, ncells, n, h->d_kp_xy[level], h->d_kp_content[level]);
    k_bucket_count<<<(n + 255) / 256, 256, 0, h->stream>>>(h->d_kp_xy[level], n, h->bw[level], h->d_bucket_tmp[level]);
  }
  k_bucket_scan<<<1, 32, 0, h->stream>>>(h->d_bucket_tmp[level], nb, h->d_bucket_ptr[level], h->d_bucket_tmp[level] + nb);
  if (n)
    k_bucket_fill<<<(n + 255) / 256, 256, 0, h->stream>>>(h->d_kp_xy[level], n, h->bw[level], h->d_bucket_tmp[level] + nb,
                                                          h->d_bucket_item[level]);
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaStreamSynchronize(h->stream));   // the FAST handle may detect again
  return SVS_OK;
}

int svs_match(svs_matcher * h, const double T_cur_from_actkey[7], const double T_actkey_from_w[7],
              const svs_match_point* pts, int n, int search_radius, int thr_mean, int thr_std, svs_match_result* out) {
  svs::NvtxRange nvtx_("match");
  if (!h || !T_cur_from_actkey || !T_actkey_from_w || n < 0 || n > h->max_pts || (n && (!pts || !out)) || search_radius < 0)
    return SVS_ERR_INVALID;
  h->last_n = 0;
  h->last_pts_own = 1;
  ++h->match_serial;
  if (n == 0) return 0;
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpyAsync(h->d_pts, pts, sizeof(svs_match_point) * (size_t)n, cudaMemcpyHostToDevice, h->stream));
  const int rc = match_launch(h, T_cur_from_actkey, T_actkey_from_w, h->d_pts, n, search_radius, thr_mean, thr_std);
  if (rc != SVS_OK) return rc;
  SVS_CK(h, cudaMemcpyAsync(out, h->d_res, sizeof(svs_match_result) * (size_t)n, cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  h->last_n = n;
  int nm = 0;
  for (int i = 0; i < n; ++i) nm += out[i].matched;
  return nm;
}

}  // extern "C"

