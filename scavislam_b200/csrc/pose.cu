// pose.cu -- motion-only Levenberg-Marquardt on sm_90a (SURVEY.md 8f rank 1, a "next" row):
// PoseOptimizer<SE3,6,IdObs<3>,3>::calcFastMotionOnly (scavislam/pose_optimizer.h:135-298) with
// SE3XYZ_STEREO (transformations.h:414-460), called after guided matching by
// StereoFrontend::matchAndTrack (stereo_frontend.cpp:1058) and Backend::globalLoopClosure
// (backend.cpp:754-779).
//
// The problem is 6 unknowns over n ~ 10^2..10^4 observations: one kernel, k_pose_lm, runs the whole
// LM loop on the device, on one CTA for up to kClusterMinObs observations and on a cluster of kCl CTAs
// above that.  A pass over the observations at pose T yields everything both the trial test and the
// next linearisation need (robust chi2, max error, J^T J, J^T f), so an accepted step costs one pass
// and a rejected step costs one pass plus a 6x6 solve; the reference recomputes A and B from the
// unchanged frame after a rejection, which gives the same numbers.  Sums are FP64, reduced in a fixed
// tree order (deterministic).  There is no host round trip inside the loop.
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>

#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include "../../include/svs_b200.h"
#include "internal.cuh"
#include "se3_dev.cuh"
#include "svs_nvtx.hpp"

namespace {

namespace cg = cooperative_groups;

constexpr int kAcc = 21 + 6 + 1;   // upper triangle of J^T J, J^T f, chi2   (max_err, norm_max_A: max-reduced)
constexpr double kEps = 0.0000000001;   // global.h:106

struct PoseCtl {
  double T[7];
  double initial_chi2, chi2, max_err;
  int num_obs, iterations, trials, nan_error;
};

struct PoseArgs {
  const int* pid;           // obs -> point index, or nullptr (identity)
  const char* obs;          // double[3] at obs + i * obs_stride
  const char* xyz;          // double[3] at xyz + pid * xyz_stride
  const char* valid;        // int at valid + i * valid_stride, or nullptr
  int obs_stride, xyz_stride, valid_stride;
  int n;
  double f, px, py, b;
  int robust, num_iter;
  double kernel_param, initial_mu, tau;
};

// pose_optimizer.h:441-449
__device__ __forceinline__ double pseudo_huber(double d, double b) {
  const double a = fabs(d);
  return a < b ? d * d : 2 * b * a - b * b;
}

struct PassOut {
  double acc[kAcc];
  double max_err, norm_max_A;
  int count;
};

// one sweep over the observations at pose (R, t)
__device__ void pass(const PoseArgs& a, const double R[9], const double t[3], PassOut& o, int first, int stride) {
#pragma unroll
  for (int k = 0; k < kAcc; ++k) o.acc[k] = 0;
  o.max_err = 0; o.norm_max_A = 0; o.count = 0;
  for (int i = first; i < a.n; i += stride) {
    if (a.valid && *reinterpret_cast<const int*>(a.valid + (size_t)i * a.valid_stride) == 0) continue;
    const int p = a.pid ? a.pid[i] : i;
    const double* X = reinterpret_cast<const double*>(a.xyz + (size_t)p * a.xyz_stride);
    const double* ob = reinterpret_cast<const double*>(a.obs + (size_t)i * a.obs_stride);
    const double X0 = X[0], X1 = X[1], X2 = X[2];
    const double x = R[0] * X0 + R[1] * X1 + R[2] * X2 + t[0];
    const double y = R[3] * X0 + R[4] * X1 + R[5] * X2 + t[1];
    const double z = R[6] * X0 + R[7] * X1 + R[8] * X2 + t[2];
    // StereoCamera::map_uvu (stereo_camera.cpp:36-44).  The divisions and square roots stay IEEE operations in the
    // reference's order: with reciprocal-multiply arithmetic (measured: the sweep is FP64-issue-bound on its one SM and
    // these are most of it) the accept/reject sequence of a nearly converged problem no longer matches the oracle's
    // (tests/test_pose_gpu.py, n = 20) -- parity first.
    double f0 = ob[0] - (a.f * (x / z) + a.px);
    double f1 = ob[1] - (a.f * (y / z) + a.py);
    double f2 = ob[2] - ((x - a.b) / z * a.f + a.px);
    if (a.robust) {
      const double nrm = fmax(kEps, sqrt(f0 * f0 + f1 * f1 + f2 * f2));
      const double w = sqrt(pseudo_huber(nrm, a.kernel_param)) / nrm;
      f0 *= w; f1 *= w; f2 *= w;
    }
    o.acc[27] += f0 * f0 + f1 * f1 + f2 * f2;
    o.max_err = fmax(o.max_err, fmax(fabs(f0), fmax(fabs(f1), fabs(f2))));
    ++o.count;
    // SE3XYZ_STEREO::frameJac (transformations.h:417-443)
    const double one_b_z = 1. / z, one_b_z_sq = 1. / (z * z);
    const double A = -a.f * one_b_z, B = -a.f * one_b_z;
    const double C = a.f * x * one_b_z_sq, D = a.f * y * one_b_z_sq, E = a.f * (x - a.b) * one_b_z_sq;
    const double J0[6] = {A, 0, C, y * C, z * A - x * C, -y * A};
    const double J1[6] = {0, B, D, -z * B + y * D, -x * D, x * B};
    const double J2[6] = {A, 0, E, y * E, z * A - x * E, -y * A};
    int k = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
#pragma unroll
      for (int c = r; c < 6; ++c) o.acc[k++] += J0[r] * J0[c] + J1[r] * J1[c] + J2[r] * J2[c];
      o.acc[21 + r] -= J0[r] * f0 + J1[r] * f1 + J2[r] * f2;
      o.norm_max_A = fmax(o.norm_max_A, fabs(J0[r] * J0[r] + J1[r] * J1[r] + J2[r] * J2[r]));
    }
  }
}

__device__ __forceinline__ double wsum(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double wmax(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <bool kCluster> struct ClusterSums {};
template <> struct ClusterSums<true> {
  double tot[kAcc + 2];   // CTA 0: sums over the cluster
  int tot_count;
};

template <int kThreads, bool kCluster>
struct Shared : ClusterSums<kCluster> {
  double part[kThreads / 32][kAcc + 2];
  int cnt[kThreads / 32];
  double sum[kAcc + 2];   // this CTA's share (on a cluster read by CTA 0 through DSMEM)
  int count;
  double R[9], t[3];      // pose under evaluation (on a cluster written by CTA 0 into every CTA)
  int go;                 // 1 = evaluate R, t; 0 = finished
  // CTA 0, thread 0: state of the LM loop, in shared memory so that it does not occupy 82 registers of every thread of the sweep
  double A[21], B[6], T[7], Tn[7];
};

// block-wide reduction of a PassOut into sh.sum / sh.count (fixed order); complete after the caller's next barrier
template <int kThreads, bool kCluster>
__device__ void reduce(Shared<kThreads, kCluster>& sh, PassOut& o) {
  constexpr int kWarps = kThreads / 32;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kAcc; ++k) {
    const double s = wsum(o.acc[k]);
    if (lane == 0) sh.part[w][k] = s;
  }
  const double me = wmax(o.max_err), na = wmax(o.norm_max_A);
  int c = o.count;
#pragma unroll
  for (int s = 16; s; s >>= 1) c += __shfl_xor_sync(0xffffffffu, c, s);
  if (lane == 0) { sh.part[w][kAcc] = me; sh.part[w][kAcc + 1] = na; sh.cnt[w] = c; }
  __syncthreads();
  if (threadIdx.x < kAcc + 2) {
    double s = 0;
    if (threadIdx.x < kAcc) for (int q = 0; q < kWarps; ++q) s += sh.part[q][threadIdx.x];
    else for (int q = 0; q < kWarps; ++q) s = fmax(s, sh.part[q][threadIdx.x]);
    sh.sum[threadIdx.x] = s;
  }
  if (threadIdx.x == 64) { int s = 0; for (int q = 0; q < kWarps; ++q) s += sh.cnt[q]; sh.count = s; }
}

// (A + mu I) x = B, A given by its upper triangle in row order (LDL^T; Eigen ldlt() in the reference)
__device__ void solve6(const double* U21, const double* B, double mu, double x[6]) {
  double A[6][6], L[6][6], D[6], y[6];
  int k = 0;
  for (int r = 0; r < 6; ++r)
    for (int c = r; c < 6; ++c) { A[r][c] = A[c][r] = U21[k++]; }
  for (int r = 0; r < 6; ++r) A[r][r] += mu;
  for (int j = 0; j < 6; ++j) {
    double d = A[j][j];
    for (int q = 0; q < j; ++q) d -= L[j][q] * L[j][q] * D[q];
    D[j] = d;
    for (int i = j + 1; i < 6; ++i) {
      double s = A[i][j];
      for (int q = 0; q < j; ++q) s -= L[i][q] * L[j][q] * D[q];
      L[i][j] = s / d;
    }
  }
  for (int i = 0; i < 6; ++i) {
    double s = B[i];
    for (int q = 0; q < i; ++q) s -= L[i][q] * y[q];
    y[i] = s;
  }
  for (int i = 5; i >= 0; --i) {
    double s = y[i] / D[i];
    for (int q = i + 1; q < 6; ++q) s -= L[q][i] * x[q];
    x[i] = s;
  }
}

// ---------------------------------------------------------------- the LM loop, on one CTA or on a thread-block cluster
// The sweep is instruction-bound on one SM (five IEEE divisions, two square roots and a 27-term accumulation per observation, kept operation for operation for parity).
// Up to kClusterMinObs observations the loop runs on one CTA of kCtaThreads threads (kCluster = false).  Above that it
// runs on a cluster of kCl CTAs of kClThreads threads, each with its own SM (kCluster = true): every CTA sweeps its share
// and reduces it in shared memory; after a cluster barrier CTA 0 adds the kCl partial results in rank order through
// distributed shared memory, its thread 0 takes the Levenberg decision and the next pose is written into every CTA's
// shared memory before the second cluster barrier of the pass.  On one CTA thread 0 reads the CTA's own sums, and there
// is neither a cluster barrier nor a pose broadcast.
constexpr int kCtaThreads = 512;
constexpr int kCl = 8;
constexpr int kClThreads = 256;
constexpr int kClusterMinObs = 512;

template <int kThreads, bool kCluster>
__global__ void __launch_bounds__(kThreads) k_pose_lm(PoseArgs a, PoseCtl* ctl) {
  using Cluster = cg::cluster_group;
  __shared__ Shared<kThreads, kCluster> sh;
  int rank = 0, nr = 1;
  if constexpr (kCluster) { rank = (int)Cluster::block_rank(); nr = (int)Cluster::num_blocks(); }
  // CTA 0, thread 0: state of the LM loop (pose_optimizer.h:142-152, 188-198)
  double mu = 0, nu = 2, chi2 = 0, max_err = 0;
  int stop = 0, trial = 0, ig = 0, iterations = 0, trials = 0;
  double* const T = sh.T; double* const Tn = sh.Tn; double* const A = sh.A; double* const B = sh.B;
  // the pose the first sweep evaluates: every CTA reads it itself
  if (threadIdx.x == 0) {
    double T0[7];
    for (int k = 0; k < 7; ++k) T0[k] = ctl->T[k];
    svs::quat_to_R(T0, sh.R);
    sh.t[0] = T0[4]; sh.t[1] = T0[5]; sh.t[2] = T0[6];
    sh.go = 1;
    if (rank == 0) for (int k = 0; k < 7; ++k) T[k] = T0[k];
  }
  __syncthreads();
  PassOut o;
  for (int sweep = 0; sh.go; ++sweep) {
    // read before the first barrier of reduce(), after which thread 0 of CTA 0 may replace it
    double R[9], t[3];
    for (int k = 0; k < 9; ++k) R[k] = sh.R[k];
    for (int k = 0; k < 3; ++k) t[k] = sh.t[k];
    pass(a, R, t, o, rank * kThreads + (int)threadIdx.x, nr * kThreads);
    reduce(sh, o);
    if constexpr (kCluster) {
      Cluster::sync();   // every CTA's share is in its sh.sum / sh.count
      if (rank == 0) {
        if (threadIdx.x < kAcc + 2) {   // fixed order: rank 0, 1, ..., nr - 1
          double s = 0;
          for (int r = 0; r < nr; ++r) {
            const double v = Cluster::map_shared_rank(sh.sum, r)[threadIdx.x];
            s = threadIdx.x < kAcc ? s + v : fmax(s, v);
          }
          sh.tot[threadIdx.x] = s;
        }
        if (threadIdx.x == 64) {
          int c = 0;
          for (int r = 0; r < nr; ++r) c += *Cluster::map_shared_rank(&sh.count, r);
          sh.tot_count = c;
        }
      }
    }
    if (rank == 0) {
      __syncthreads();
      if (threadIdx.x == 0) {
        const double* tot;
        int num;
        if constexpr (kCluster) { tot = sh.tot; num = sh.tot_count; } else { tot = sh.sum; num = sh.count; }
        int go = 0;
        if (sweep == 0) {   // pose_optimizer.h:142-152, 188-198
          for (int k = 0; k < 21; ++k) A[k] = tot[k];
          for (int k = 0; k < 6; ++k) B[k] = tot[21 + k];
          chi2 = tot[27]; max_err = tot[kAcc];
          ctl->initial_chi2 = chi2; ctl->num_obs = num; ctl->nan_error = 0;
          mu = a.initial_mu == -1 ? a.tau * tot[kAcc + 1] : a.initial_mu;
          go = (a.num_iter > 0 && num > 0) ? 1 : 0;
        } else {
          const double new_chi2 = tot[27];
          ++trials;
          bool next_iter = false;
          if (isnan(new_chi2)) {            // the reference throws (pose_optimizer.h:265-268)
            ctl->nan_error = 1; stop = 1;
          } else {
            const double rho = chi2 - new_chi2;
            if (rho > 0) {                  // :270-278
              for (int k = 0; k < 7; ++k) T[k] = Tn[k];
              chi2 = new_chi2; max_err = tot[kAcc];
              double nb = 0;
              for (int k = 0; k < 6; ++k) nb = fmax(nb, fabs(B[k]));
              stop = nb <= kEps;
              const double c = 2 * rho - 1;
              mu *= fmax(1. / 3., 1 - c * c * c);
              nu = 2.; trial = 0; ++iterations;
              for (int k = 0; k < 21; ++k) A[k] = tot[k];
              for (int k = 0; k < 6; ++k) B[k] = tot[21 + k];
              next_iter = true;
            } else {                        // :280-293
              mu *= nu; nu *= 2.; ++trial;
              if (trial == 5) stop = 1;
            }
          }
          if (next_iter) ++ig;
          go = (stop || (next_iter && ig >= a.num_iter)) ? 0 : 1;
        }
        if (go) {
          double x[6], dT[7];
          solve6(A, B, mu, x);
          svs::se3_exp(x, dT);              // SE3_AbstractPoint::add (transformations.h:408-411)
          svs::se3_mul(dT, T, Tn);
          svs::quat_to_R(Tn, sh.R);
          sh.t[0] = Tn[4]; sh.t[1] = Tn[5]; sh.t[2] = Tn[6];
        }
        sh.go = go;
      }
      __syncthreads();
      if constexpr (kCluster) {
        // the next pose (or the end) goes into every other CTA's shared memory
        for (int i = threadIdx.x; i < (nr - 1) * 13; i += kThreads) {
          const int r = 1 + i / 13, q = i - (r - 1) * 13;
          if (q < 9) Cluster::map_shared_rank(sh.R, r)[q] = sh.R[q];
          else if (q < 12) Cluster::map_shared_rank(sh.t, r)[q - 9] = sh.t[q - 9];
          else *Cluster::map_shared_rank(&sh.go, r) = sh.go;
        }
      }
    }
    if constexpr (kCluster) Cluster::sync();   // the pose of the next sweep is in place; nobody reads a remote sh.sum any more
  }
  if (rank == 0 && threadIdx.x == 0) {
    for (int k = 0; k < 7; ++k) ctl->T[k] = T[k];
    ctl->chi2 = chi2; ctl->max_err = max_err; ctl->iterations = iterations; ctl->trials = trials;
  }
}

}  // namespace

struct svs_pose {
  int device = 0, max_obs = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  std::string err;
  int* d_pid = nullptr;
  double* d_obs = nullptr;
  double* d_xyz = nullptr;
  PoseCtl* d_ctl = nullptr;
  PoseCtl* h_ctl = nullptr;   // pinned
};

#define QCK(call)                                                       \
  do {                                                                  \
    cudaError_t e_ = (call);                                            \
    if (e_ != cudaSuccess) {                                            \
      h->err = std::string(#call) + ": " + cudaGetErrorString(e_);      \
      return SVS_ERR_CUDA;                                              \
    }                                                                   \
  } while (0)

static int run(svs_pose* h, PoseArgs& a, const svs_cam* cam, const svs_pose_params* p, double T[7],
               svs_pose_stats* stats) {
  a.f = cam->f; a.px = cam->px; a.py = cam->py; a.b = cam->b;
  a.robust = p->robust_kernel; a.num_iter = p->num_iter; a.kernel_param = p->kernel_param;
  a.initial_mu = p->initial_mu; a.tau = p->tau;
  memcpy(h->h_ctl->T, T, sizeof(double) * 7);
  QCK(cudaMemcpyAsync(h->d_ctl, h->h_ctl, sizeof(double) * 7, cudaMemcpyHostToDevice, h->stream));
  QCK(cudaEventRecord(h->ev0, h->stream));
  if (a.n > kClusterMinObs) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(kCl, 1, 1);
    cfg.blockDim = dim3(kClThreads, 1, 1);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = h->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = kCl; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if (cudaLaunchKernelEx(&cfg, k_pose_lm<kClThreads, true>, a, h->d_ctl) != cudaSuccess) {
      (void)cudaGetLastError();   // a partition that cannot co-schedule eight CTAs: the one-CTA shape computes the same
      k_pose_lm<kCtaThreads, false><<<1, kCtaThreads, 0, h->stream>>>(a, h->d_ctl);
    }
  } else {
    k_pose_lm<kCtaThreads, false><<<1, kCtaThreads, 0, h->stream>>>(a, h->d_ctl);
  }
  QCK(cudaGetLastError());
  QCK(cudaEventRecord(h->ev1, h->stream));
  QCK(cudaMemcpyAsync(h->h_ctl, h->d_ctl, sizeof(PoseCtl), cudaMemcpyDeviceToHost, h->stream));
  QCK(cudaStreamSynchronize(h->stream));
  const PoseCtl& c = *h->h_ctl;
  if (c.nan_error) { h->err = "Res is NaN!"; return SVS_ERR_NUMERIC; }
  memcpy(T, c.T, sizeof(double) * 7);
  if (stats) {
    stats->initial_chi2 = c.initial_chi2; stats->chi2 = c.chi2; stats->max_err = c.max_err;
    stats->num_obs = c.num_obs; stats->iterations = c.iterations; stats->trials = c.trials;
    float ms = 0; cudaEventElapsedTime(&ms, h->ev0, h->ev1); stats->ms = ms;
  }
  return SVS_OK;
}

extern "C" {

int svs_pose_create(int device, int max_obs, svs_pose** out) {
  if (!out || max_obs <= 0) return SVS_ERR_INVALID;
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return SVS_ERR_NOGPU;
  svs_pose* h = new svs_pose();
  if (device < 0) cudaGetDevice(&device);
  h->device = device; h->max_obs = max_obs;
  const bool ok = cudaSetDevice(device) == cudaSuccess &&
                  cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) == cudaSuccess &&
                  cudaEventCreate(&h->ev0) == cudaSuccess && cudaEventCreate(&h->ev1) == cudaSuccess &&
                  cudaMalloc(&h->d_pid, sizeof(int) * (size_t)max_obs) == cudaSuccess &&
                  cudaMalloc(&h->d_obs, sizeof(double) * 3 * (size_t)max_obs) == cudaSuccess &&
                  cudaMalloc(&h->d_xyz, sizeof(double) * 3 * (size_t)max_obs) == cudaSuccess &&
                  cudaMalloc(&h->d_ctl, sizeof(PoseCtl)) == cudaSuccess &&
                  cudaMallocHost(&h->h_ctl, sizeof(PoseCtl)) == cudaSuccess;
  if (!ok) { svs_pose_destroy(h); return SVS_ERR_CUDA; }
  *out = h;
  return SVS_OK;
}

void svs_pose_destroy(svs_pose* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  cudaFree(h->d_pid); cudaFree(h->d_obs); cudaFree(h->d_xyz); cudaFree(h->d_ctl);
  if (h->h_ctl) cudaFreeHost(h->h_ctl);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

const char* svs_pose_last_error(const svs_pose* h) { return h ? h->err.c_str() : "null handle"; }

int svs_calcFastMotionOnly(svs_pose* h, int n, const int* obs_point_id, const double* obs_uvu, int npoints,
                           const double* point_xyz, const svs_cam* cam, const svs_pose_params* params, double T_frame[7],
                           svs_pose_stats* stats) {
  svs::NvtxRange nvtx_("match");
  if (!h || n <= 0 || !obs_point_id || !obs_uvu || npoints <= 0 || !point_xyz || !cam || !params || !T_frame)
    return SVS_ERR_INVALID;                       // the reference asserts obs_list.size() > 0
  if (n > h->max_obs || npoints > h->max_obs) { h->err = "more observations/points than the handle's capacity"; return SVS_ERR_INVALID; }
  for (int i = 0; i < n; ++i)
    if (obs_point_id[i] < 0 || obs_point_id[i] >= npoints) { h->err = "obs.point_id outside point_list"; return SVS_ERR_INVALID; }
  cudaSetDevice(h->device);
  QCK(cudaMemcpyAsync(h->d_pid, obs_point_id, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, h->stream));
  QCK(cudaMemcpyAsync(h->d_obs, obs_uvu, sizeof(double) * 3 * (size_t)n, cudaMemcpyHostToDevice, h->stream));
  QCK(cudaMemcpyAsync(h->d_xyz, point_xyz, sizeof(double) * 3 * (size_t)npoints, cudaMemcpyHostToDevice, h->stream));
  PoseArgs a;
  memset(&a, 0, sizeof a);
  a.pid = h->d_pid; a.obs = reinterpret_cast<const char*>(h->d_obs); a.xyz = reinterpret_cast<const char*>(h->d_xyz);
  a.obs_stride = a.xyz_stride = 3 * sizeof(double); a.n = n;
  return run(h, a, cam, params, T_frame, stats);
}

int svs_calcFastMotionOnly_matched(svs_pose* h, svs_matcher* m, const svs_cam* cam, const svs_pose_params* params,
                                   double T_frame[7], svs_pose_stats* stats) {
  svs::NvtxRange nvtx_("match");
  if (!h || !m || !cam || !params || !T_frame) return SVS_ERR_INVALID;
  const svs_match_result* d_res = nullptr;
  int n = 0, dev = -1;
  svs::matcher_device_results(m, &d_res, &n, &dev);
  if (dev != h->device) { h->err = "matcher lives on another device"; return SVS_ERR_INVALID; }
  if (n <= 0 || !d_res) { h->err = "no svs_match results on the device"; return SVS_ERR_STATE; }
  cudaSetDevice(h->device);
  PoseArgs a;
  memset(&a, 0, sizeof a);
  const char* base = reinterpret_cast<const char*>(d_res);
  a.obs = base + offsetof(svs_match_result, obs);
  a.xyz = base + offsetof(svs_match_result, xyz_actkey);
  a.valid = base + offsetof(svs_match_result, matched);
  a.obs_stride = a.xyz_stride = a.valid_stride = sizeof(svs_match_result);
  a.n = n;
  return run(h, a, cam, params, T_frame, stats);   // svs_match has synchronised its stream
}

}  // extern "C"
