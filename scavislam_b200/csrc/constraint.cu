// constraint.cu -- SlamGraph::computeConstraint (scavislam/slam_graph.cpp:785-846) batched over pose pairs
// (SURVEY.md 8f rank 4, a "next" row): relative pose T_1_from_2, the median distance of the landmarks both
// frames observe, and the information matrix Lambda = n diag((350 |t| / median)^2 I3, 100^2 I3) the
// pose-pose edges of the double window carry (a11).  Called per edge on marginalisation and key-frame
// insertion (slam_graph.cpp:848-904).
//
// One CTA per pair: the threads walk the shorter... v1's feature table and look every point up in v2's by
// binary search (both tables ascending by point id), transform the shared ones into frame 1 and collect
// their distances; the median is taken by rank counting (exact multiset median, maths_utils.h:113-136),
// in shared memory when the pair shares <= 2048 points, in a global scratch row otherwise.
#include <cmath>
#include <cstring>
#include <string>

#include <cuda_runtime.h>

#include "../../include/svs_b200.h"
#include "handle.cuh"
#include "internal.cuh"
#include "se3_dev.cuh"

namespace {

constexpr int kThreads = 128;
constexpr int kSmemDepths = 2048;

struct CArgs {
  const double* poses;
  const int* feat_ptr;
  const int* feat_point;
  const int* point_anchor;
  const double* xyz;
  const int* v1;
  const int* v2;
  double* T12;
  double* Lambda;
  int* strength;
  double* scratch;     // [npairs][scratch_stride]
  int scratch_stride;
};

__global__ void __launch_bounds__(kThreads) k_compute_constraint(CArgs a) {
  __shared__ double sDepth[kSmemDepths];
  __shared__ double sT1[7], sT12[7], sMed[2];
  __shared__ int sCount;
  const int k = blockIdx.x;
  const int p1 = a.v1[k], p2 = a.v2[k];
  if (threadIdx.x == 0) {
    double T2i[7];
    for (int q = 0; q < 7; ++q) sT1[q] = a.poses[7 * (size_t)p1 + q];
    svs::se3_inv(a.poses + 7 * (size_t)p2, T2i);
    svs::se3_mul(sT1, T2i, sT12);          // slam_graph.cpp:793
    sCount = 0; sMed[0] = sMed[1] = 0.;
  }
  __syncthreads();
  const int a0 = a.feat_ptr[p1], a1 = a.feat_ptr[p1 + 1], b0 = a.feat_ptr[p2], b1 = a.feat_ptr[p2 + 1];
  const bool in_smem = min(a1 - a0, b1 - b0) <= kSmemDepths;
  double* depth = in_smem ? sDepth : a.scratch + (size_t)k * a.scratch_stride;
  for (int i = a0 + (int)threadIdx.x; i < a1; i += kThreads) {
    const int p = a.feat_point[i];
    int lo = b0, hi = b1;                  // v2.feature_table.find(point_id)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (a.feat_point[mid] < p) lo = mid + 1; else hi = mid;
    }
    if (lo >= b1 || a.feat_point[lo] != p) continue;
    double Tai[7], A[7], T1[7];
    for (int q = 0; q < 7; ++q) T1[q] = sT1[q];
    svs::se3_inv(a.poses + 7 * (size_t)a.point_anchor[p], Tai);
    svs::se3_mul(T1, Tai, A);              // v1.T_me_from_world * T_anchor_from_w.inverse() * p.xyz_anchor (:826-829)
    double R[9], x[3];
    svs::quat_to_R(A, R);
    svs::mat3_vec(R, a.xyz + 3 * (size_t)p, x);
    x[0] += A[4]; x[1] += A[5]; x[2] += A[6];
    depth[atomicAdd(&sCount, 1)] = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
  }
  __threadfence_block();
  __syncthreads();
  const int n = sCount;
  // exact multiset median by rank counting (order of insertion does not matter: equal values are interchangeable)
  const int r_hi = n / 2, r_lo = (n % 2) ? n / 2 : n / 2 - 1;
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const double di = depth[i];
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      const double dj = depth[j];
      rank += (dj < di) || (dj == di && j < i);
    }
    if (rank == r_lo) sMed[0] = di;
    if (rank == r_hi) sMed[1] = di;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 0; q < 7; ++q) a.T12[7 * (size_t)k + q] = sT12[q];
    a.strength[k] = n;
  }
  if (threadIdx.x < 36) {
    double v = 0.;
    const int r = threadIdx.x / 6, c = threadIdx.x - 6 * r;
    if (n > 0 && r == c) {
      const double med = (n % 2) ? sMed[1] : 0.5 * (sMed[0] + sMed[1]);
      const double nd = sqrt(sT12[4] * sT12[4] + sT12[5] * sT12[5] + sT12[6] * sT12[6]) / med;   // :840-841
      const double s = r < 3 ? 350 * 1. * nd : 100 * 1.;
      v = (double)n * (s * s);                                                                 // :843-846
    }
    a.Lambda[36 * (size_t)k + threadIdx.x] = v;
  }
}

}  // namespace

int svs::constraint_scratch_stride(int max_feat) { return max_feat > kSmemDepths ? max_feat : 0; }

void svs::launch_compute_constraint(const double* poses, const int* feat_ptr, const int* feat_point, const int* point_anchor,
                                    const double* xyz, int npairs, const int* v1, const int* v2, double* T_1_from_2,
                                    double* Lambda, int* strength, double* scratch, int scratch_stride, cudaStream_t stream) {
  CArgs a;
  a.poses = poses; a.feat_ptr = feat_ptr; a.feat_point = feat_point; a.point_anchor = point_anchor; a.xyz = xyz;
  a.v1 = v1; a.v2 = v2; a.T12 = T_1_from_2; a.Lambda = Lambda; a.strength = strength;
  a.scratch = scratch; a.scratch_stride = scratch_stride;
  k_compute_constraint<<<npairs, kThreads, 0, stream>>>(a);
}

struct svs_constraints : svs::Handle {
  size_t cap_bytes = 0;
  char* d_buf = nullptr;
};

extern "C" {

int svs_constraints_create(int device, svs_constraints** out) {
  if (!out) return SVS_ERR_INVALID;
  *out = nullptr;
  svs_constraints* h = new svs_constraints();
  if (int rc = svs::open_handle(h, device)) {
    delete h;
    return rc;
  }
  *out = h;
  return SVS_OK;
}

void svs_constraints_destroy(svs_constraints* h) {
  if (!h) return;
  svs::begin_close(h);
  cudaFree(h->d_buf);
  delete h;
}

const char* svs_constraints_last_error(const svs_constraints* h) { return svs::last_error(h); }

int svs_computeConstraint_batch(svs_constraints* h, int P, const double* T_me_from_world, const int* feat_ptr,
                                const int* feat_point, int L, const int* point_anchor, const double* xyz_anchor, int npairs,
                                const int* v1, const int* v2, double* T_1_from_2, double* Lambda, int* visibility_strength) {
  if (!h || P <= 0 || !T_me_from_world || !feat_ptr || L < 0 || npairs < 0 || (npairs && (!v1 || !v2 || !T_1_from_2 || !Lambda)))
    return SVS_ERR_INVALID;
  if (npairs == 0) return SVS_OK;
  const int nfeat = feat_ptr[P];
  if (nfeat < 0 || (nfeat && !feat_point) || (L && (!point_anchor || !xyz_anchor))) return SVS_ERR_INVALID;
  int max_feat = 0;
  for (int p = 0; p < P; ++p) {
    if (feat_ptr[p + 1] < feat_ptr[p]) { h->err = "feat_ptr not ascending"; return SVS_ERR_INVALID; }
    max_feat = std::max(max_feat, feat_ptr[p + 1] - feat_ptr[p]);
    for (int i = feat_ptr[p]; i < feat_ptr[p + 1]; ++i) {
      if (feat_point[i] < 0 || feat_point[i] >= L) { h->err = "feature names a point outside [0, L)"; return SVS_ERR_INVALID; }
      if (i > feat_ptr[p] && feat_point[i] <= feat_point[i - 1]) { h->err = "feature table not strictly ascending by point id"; return SVS_ERR_INVALID; }
    }
  }
  for (int l = 0; l < L; ++l)
    if (point_anchor[l] < 0 || point_anchor[l] >= P) { h->err = "point anchored in a frame outside [0, P)"; return SVS_ERR_INVALID; }
  for (int k = 0; k < npairs; ++k)
    if (v1[k] < 0 || v1[k] >= P || v2[k] < 0 || v2[k] >= P) { h->err = "pair names a pose outside [0, P)"; return SVS_ERR_INVALID; }
  cudaSetDevice(h->device);
  const int scratch_stride = svs::constraint_scratch_stride(max_feat);
  // one arena: inputs, outputs, scratch
  struct {
    double *pose, *xyz, *T12, *Lam, *scr;
    int *fptr, *fpt, *anch, *v1, *v2, *n;
  } b;
  auto carve = [&](svs::Bump m) {
    b.pose = m.take<double>(7 * (size_t)P); b.fptr = m.take<int>((size_t)P + 1); b.fpt = m.take<int>(nfeat);
    b.anch = m.take<int>(L); b.xyz = m.take<double>(3 * (size_t)L);
    b.v1 = m.take<int>(npairs); b.v2 = m.take<int>(npairs); b.T12 = m.take<double>(7 * (size_t)npairs);
    b.Lam = m.take<double>(36 * (size_t)npairs); b.n = m.take<int>(npairs);
    b.scr = m.take<double>((size_t)scratch_stride * npairs);
    return m.off;
  };
  const size_t bytes = carve(svs::Bump{nullptr});
  if (bytes > h->cap_bytes) {
    SVS_CK(h, cudaStreamSynchronize(h->stream));
    SVS_CK(h, svs::grow(bytes, &h->cap_bytes, &h->d_buf));
  }
  carve(svs::Bump{h->d_buf});
  SVS_CK(h, cudaMemcpyAsync(b.pose, T_me_from_world, sizeof(double) * 7 * (size_t)P, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaMemcpyAsync(b.fptr, feat_ptr, sizeof(int) * ((size_t)P + 1), cudaMemcpyHostToDevice, h->stream));
  if (nfeat) SVS_CK(h, cudaMemcpyAsync(b.fpt, feat_point, sizeof(int) * (size_t)nfeat, cudaMemcpyHostToDevice, h->stream));
  if (L) {
    SVS_CK(h, cudaMemcpyAsync(b.anch, point_anchor, sizeof(int) * (size_t)L, cudaMemcpyHostToDevice, h->stream));
    SVS_CK(h, cudaMemcpyAsync(b.xyz, xyz_anchor, sizeof(double) * 3 * (size_t)L, cudaMemcpyHostToDevice, h->stream));
  }
  SVS_CK(h, cudaMemcpyAsync(b.v1, v1, sizeof(int) * (size_t)npairs, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaMemcpyAsync(b.v2, v2, sizeof(int) * (size_t)npairs, cudaMemcpyHostToDevice, h->stream));
  svs::launch_compute_constraint(b.pose, b.fptr, b.fpt, b.anch, b.xyz, npairs, b.v1, b.v2, b.T12, b.Lam, b.n, b.scr,
                                 scratch_stride, h->stream);
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaMemcpyAsync(T_1_from_2, b.T12, sizeof(double) * 7 * (size_t)npairs, cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaMemcpyAsync(Lambda, b.Lam, sizeof(double) * 36 * (size_t)npairs, cudaMemcpyDeviceToHost, h->stream));
  if (visibility_strength)
    SVS_CK(h, cudaMemcpyAsync(visibility_strength, b.n, sizeof(int) * (size_t)npairs, cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  return SVS_OK;
}

}  // extern "C"
