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
//
// svs_calcFastMotionOnly_device runs the same kernel on a track handed over in GPU memory; svs_pose_grad differentiates
// the returned pose with respect to the observations, points and camera (the kernels after k_pose_lm).
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>

#include <cooperative_groups.h>
#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "../../include/svs_b200.h"
#include "handle.cuh"
#include "internal.cuh"
#include "se3_dev.cuh"
#include "svs_nvtx.hpp"

namespace {

namespace cg = cooperative_groups;

constexpr int kAcc = 21 + 6 + 1;   // upper triangle of J^T J, J^T f, chi2   (max_err, norm_max_A: max-reduced)
constexpr double kEps = 0.0000000001;   // global.h:106

struct PoseCtl {
  double T[7];
  int bad_pid;   // device input: some obs.point_id lies outside [0, npoints) (k_pose_ingest); uploaded with T
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

// Device input: obs.point_id into the handle's buffer, an id outside [0, npoints) flagged in ctl->bad_pid and replaced
// by 0 so that the LM kernel that follows on the stream reads only inside point_list (its result is then discarded).
__global__ void __launch_bounds__(256) k_pose_ingest(const int* __restrict__ src, int n, int npoints, int* __restrict__ dst,
                                                     PoseCtl* ctl) {
  const int i = (int)(blockIdx.x * 256u + threadIdx.x);
  if (i >= n) return;
  const int p = src[i];
  const bool bad = p < 0 || p >= npoints;
  dst[i] = bad ? 0 : p;
  if (bad) ctl->bad_pid = 1;
}

// ---------------------------------------------------------------- svs_pose_grad: the derivative of the LM's root
// The pose the LM returns is the root of F(T) = sum_i J_i^T w_i f_i (its normal equations' right-hand side), with
// f_i = z_i - pi(T X_{p_i}) and w_i = sqrt(rho(r_i)) / r_i the pseudo-Huber reweighting.  Implicit differentiation,
// dropping the derivatives of J_i (Gauss-Newton): H = sum_i J_i^T W_i J_i with W_i = d(w_i f_i)/df_i, v = (H + lambda I)^-1 g,
// u_i = W_i J_i v, and then dL/dz_i = -u_i, dL/dX_p = sum_{i: p_i = p} (dpi_i/dX)^T u_i, dL/dcam = sum_i (dpi_i/dcam)^T u_i.
//   k_pose_grad_h       H at T* on the forward's launch shape, then (H + lambda I) v = g by Cholesky with a
//                       positive-definiteness test (one thread)
//   k_pose_grad_obs     one thread per observation: dL/dz_i, and its point and camera partials
//   k_pose_grad_points  one thread per point: its partials in ascending observation order (a stable sort by point)
//   k_pose_grad_cam     one CTA: the camera partials in a fixed order
// Every sum runs in a fixed order without atomics: repeated calls give the same bits.

struct PoseGradCtl {
  double g[6];          // dL/d delta from host memory
  double v[6];          // (H + lambda I)^-1 g
  double R[9], t[3];    // T* as the forward's last sweep evaluated it
  int fail;             // H + lambda I not positive definite
};

// Observation i at (R, t): the point in the camera, f (unweighted), J = df/d delta and W = w (I - c f f^T)
struct ObsLin {
  double x, y, z, f[3], J0[6], J1[6], J2[6], w, c;
};

__device__ __forceinline__ void linearise(const PoseArgs& a, const double R[9], const double t[3], int i, ObsLin& o) {
  const int p = a.pid ? a.pid[i] : i;
  const double* X = reinterpret_cast<const double*>(a.xyz + (size_t)p * a.xyz_stride);
  const double* ob = reinterpret_cast<const double*>(a.obs + (size_t)i * a.obs_stride);
  const double X0 = X[0], X1 = X[1], X2 = X[2];
  const double x = R[0] * X0 + R[1] * X1 + R[2] * X2 + t[0];
  const double y = R[3] * X0 + R[4] * X1 + R[5] * X2 + t[1];
  const double z = R[6] * X0 + R[7] * X1 + R[8] * X2 + t[2];
  o.x = x; o.y = y; o.z = z;
  o.f[0] = ob[0] - (a.f * (x / z) + a.px);
  o.f[1] = ob[1] - (a.f * (y / z) + a.py);
  o.f[2] = ob[2] - ((x - a.b) / z * a.f + a.px);
  // d(w f)/df: w = 1 inside the kernel's quadratic branch; beyond it (r >= b) w = sqrt(2 b r - b^2) / r and
  // W = w (I - (r - b) / (2 r - b) f^ f^T), written with the unnormalised f: c = (r - b) / ((2 r - b) r^2)
  o.w = 1; o.c = 0;
  if (a.robust) {
    const double r = fmax(kEps, sqrt(o.f[0] * o.f[0] + o.f[1] * o.f[1] + o.f[2] * o.f[2]));
    const double b = a.kernel_param;
    if (!(r < b)) {
      o.w = sqrt(pseudo_huber(r, b)) / r;
      o.c = (r - b) / ((2 * r - b) * r * r);
    }
  }
  // SE3XYZ_STEREO::frameJac, as in pass()
  const double one_b_z = 1. / z, one_b_z_sq = 1. / (z * z);
  const double A = -a.f * one_b_z, B = -a.f * one_b_z;
  const double C = a.f * x * one_b_z_sq, D = a.f * y * one_b_z_sq, E = a.f * (x - a.b) * one_b_z_sq;
  const double J0[6] = {A, 0, C, y * C, z * A - x * C, -y * A};
  const double J1[6] = {0, B, D, -z * B + y * D, -x * D, x * B};
  const double J2[6] = {A, 0, E, y * E, z * A - x * E, -y * A};
#pragma unroll
  for (int k = 0; k < 6; ++k) { o.J0[k] = J0[k]; o.J1[k] = J1[k]; o.J2[k] = J2[k]; }
}

// e <- W e
__device__ __forceinline__ void apply_w(const ObsLin& o, double e[3]) {
  const double fe = o.c * (o.f[0] * e[0] + o.f[1] * e[1] + o.f[2] * e[2]);
#pragma unroll
  for (int k = 0; k < 3; ++k) e[k] = o.w * (e[k] - fe * o.f[k]);
}

// (U + lambda I) v = g, U given by its upper triangle in row order, by Cholesky; false when not positive definite
__device__ bool chol_solve6(const double* U21, double lambda, const double* g, double v[6]) {
  double A[6][6], L[6][6], y[6];
  int k = 0;
  for (int r = 0; r < 6; ++r)
    for (int c = r; c < 6; ++c) { A[r][c] = A[c][r] = U21[k++]; }
  for (int r = 0; r < 6; ++r) A[r][r] += lambda;
  for (int j = 0; j < 6; ++j) {
    double d = A[j][j];
    for (int q = 0; q < j; ++q) d -= L[j][q] * L[j][q];
    if (!(d > 0)) return false;      // also NaN
    L[j][j] = sqrt(d);
    for (int i = j + 1; i < 6; ++i) {
      double s = A[i][j];
      for (int q = 0; q < j; ++q) s -= L[i][q] * L[j][q];
      L[i][j] = s / L[j][j];
    }
  }
  for (int i = 0; i < 6; ++i) {
    double s = g ? g[i] : 0.;
    for (int q = 0; q < i; ++q) s -= L[i][q] * y[q];
    y[i] = s / L[i][i];
  }
  for (int i = 5; i >= 0; --i) {
    double s = y[i];
    for (int q = i + 1; q < 6; ++q) s -= L[q][i] * v[q];
    v[i] = s / L[i][i];
  }
  bool finite = true;
  for (int i = 0; i < 6; ++i) finite = finite && isfinite(v[i]);
  return finite;
}

template <int kThreads, bool kCluster>
struct GradShared {
  double part[kThreads / 32][21];
  double sum[21];   // this CTA's share (on a cluster read by CTA 0 through DSMEM)
  double tot[21];
  double R[9], t[3];
};

// H at T* summed as k_pose_lm sums J^T J (one CTA, or kCl CTAs added in rank order), then the solve on CTA 0, thread 0
template <int kThreads, bool kCluster>
__global__ void __launch_bounds__(kThreads) k_pose_grad_h(PoseArgs a, const PoseCtl* ctl, const double* g, double lambda,
                                                          PoseGradCtl* gc) {
  using Cluster = cg::cluster_group;
  constexpr int kWarps = kThreads / 32;
  __shared__ GradShared<kThreads, kCluster> sh;
  int rank = 0, nr = 1;
  if constexpr (kCluster) { rank = (int)Cluster::block_rank(); nr = (int)Cluster::num_blocks(); }
  if (threadIdx.x == 0) {
    double T[7];
    for (int k = 0; k < 7; ++k) T[k] = ctl->T[k];
    svs::quat_to_R(T, sh.R);
    sh.t[0] = T[4]; sh.t[1] = T[5]; sh.t[2] = T[6];
  }
  __syncthreads();
  double R[9], t[3];
  for (int k = 0; k < 9; ++k) R[k] = sh.R[k];
  for (int k = 0; k < 3; ++k) t[k] = sh.t[k];
  double acc[21];
#pragma unroll
  for (int k = 0; k < 21; ++k) acc[k] = 0;
  for (int i = rank * kThreads + (int)threadIdx.x; i < a.n; i += nr * kThreads) {
    ObsLin o;
    linearise(a, R, t, i, o);
    double M0[6], M1[6], M2[6];   // W J, column by column
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      double e[3] = {o.J0[c], o.J1[c], o.J2[c]};
      apply_w(o, e);
      M0[c] = e[0]; M1[c] = e[1]; M2[c] = e[2];
    }
    int k = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r)
#pragma unroll
      for (int c = r; c < 6; ++c) acc[k++] += o.J0[r] * M0[c] + o.J1[r] * M1[c] + o.J2[r] * M2[c];
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 21; ++k) {
    const double s = wsum(acc[k]);
    if (lane == 0) sh.part[w][k] = s;
  }
  __syncthreads();
  if (threadIdx.x < 21) {
    double s = 0;
    for (int q = 0; q < kWarps; ++q) s += sh.part[q][threadIdx.x];
    sh.sum[threadIdx.x] = s;
  }
  const double* tot = sh.sum;
  if constexpr (kCluster) {
    Cluster::sync();   // every CTA's share is in its sh.sum
    if (rank == 0 && threadIdx.x < 21) {   // fixed order: rank 0, 1, ..., nr - 1
      double s = 0;
      for (int r = 0; r < nr; ++r) s += Cluster::map_shared_rank(sh.sum, r)[threadIdx.x];
      sh.tot[threadIdx.x] = s;
    }
    tot = sh.tot;
  }
  __syncthreads();
  if (rank == 0 && threadIdx.x == 0) {
    double v[6];
    const bool ok = chol_solve6(tot, lambda, g, v);
    for (int k = 0; k < 6; ++k) gc->v[k] = ok ? v[k] : 0.;
    for (int k = 0; k < 9; ++k) gc->R[k] = R[k];
    for (int k = 0; k < 3; ++k) gc->t[k] = t[k];
    gc->fail = ok ? 0 : 1;
  }
  if constexpr (kCluster) Cluster::sync();   // nobody reads a remote sh.sum any more
}

constexpr int kGradThreads = 256;

// One thread per observation: u = W J v; dobs[i] = -u, the point partial q[i] = (dpi/dX)^T u = R^T (dpi/dy)^T u and
// the camera partial c[i] = (dpi/d(f, px, py, b))^T u (any of the three may be nullptr)
__global__ void __launch_bounds__(kGradThreads) k_pose_grad_obs(PoseArgs a, const PoseGradCtl* __restrict__ gc,
                                                                double* __restrict__ dobs, double* __restrict__ q,
                                                                double* __restrict__ c) {
  const int i = (int)(blockIdx.x * (unsigned)kGradThreads + threadIdx.x);
  if (i >= a.n) return;
  double R[9], t[3], v[6];
  for (int k = 0; k < 9; ++k) R[k] = gc->R[k];
  for (int k = 0; k < 3; ++k) t[k] = gc->t[k];
  for (int k = 0; k < 6; ++k) v[k] = gc->v[k];
  const bool fail = gc->fail != 0;
  ObsLin o;
  linearise(a, R, t, i, o);
  double u[3] = {0, 0, 0};
#pragma unroll
  for (int k = 0; k < 6; ++k) { u[0] += o.J0[k] * v[k]; u[1] += o.J1[k] * v[k]; u[2] += o.J2[k] * v[k]; }
  apply_w(o, u);
  if (dobs)
#pragma unroll
    for (int k = 0; k < 3; ++k) dobs[3 * (size_t)i + k] = fail ? 0. : -u[k];
  const double iz = 1. / o.z;
  if (q) {
    // dpi/dy = -J[:, 0:3]
    const double gy[3] = {-(o.J0[0] * u[0] + o.J2[0] * u[2]), -(o.J1[1] * u[1]),
                          -(o.J0[2] * u[0] + o.J1[2] * u[1] + o.J2[2] * u[2])};
#pragma unroll
    for (int k = 0; k < 3; ++k) q[3 * (size_t)i + k] = R[k] * gy[0] + R[3 + k] * gy[1] + R[6 + k] * gy[2];
  }
  if (c) {
    c[4 * (size_t)i + 0] = (o.x * u[0] + o.y * u[1] + (o.x - a.b) * u[2]) * iz;
    c[4 * (size_t)i + 1] = u[0] + u[2];
    c[4 * (size_t)i + 2] = u[1];
    c[4 * (size_t)i + 3] = -a.f * iz * u[2];
  }
}

// One thread per point: the partials of its observations in ascending observation order
__global__ void __launch_bounds__(kGradThreads) k_pose_grad_points(const int* __restrict__ order, const int* __restrict__ start,
                                                                   const int* __restrict__ end, const double* __restrict__ q,
                                                                   int npoints, const PoseGradCtl* __restrict__ gc,
                                                                   double* __restrict__ dxyz) {
  const int p = (int)(blockIdx.x * (unsigned)kGradThreads + threadIdx.x);
  if (p >= npoints) return;
  double s[3] = {0, 0, 0};
  for (int k = start[p]; k < end[p]; ++k) {
    const int i = order[k];
#pragma unroll
    for (int j = 0; j < 3; ++j) s[j] += q[3 * (size_t)i + j];
  }
  const bool fail = gc->fail != 0;
#pragma unroll
  for (int j = 0; j < 3; ++j) dxyz[3 * (size_t)p + j] = fail ? 0. : s[j];
}

// One CTA: out[k] = sum over observations of c[i][k], each thread over a fixed stride, then a fixed tree
__global__ void __launch_bounds__(kGradThreads) k_pose_grad_cam(const double* __restrict__ c, int n,
                                                                const PoseGradCtl* __restrict__ gc, double* __restrict__ out) {
  __shared__ double sh[4][kGradThreads];
  const int t = threadIdx.x;
  double s[4] = {0., 0., 0., 0.};
  for (int i = t; i < n; i += kGradThreads)
#pragma unroll
    for (int k = 0; k < 4; ++k) s[k] += c[4 * (size_t)i + k];
#pragma unroll
  for (int k = 0; k < 4; ++k) sh[k][t] = s[k];
  __syncthreads();
  for (int w = kGradThreads / 2; w > 0; w >>= 1) {
    if (t < w)
#pragma unroll
      for (int k = 0; k < 4; ++k) sh[k][t] += sh[k][t + w];
    __syncthreads();
  }
  if (t < 4) out[t] = gc->fail ? 0. : sh[t][0];
}

__global__ void __launch_bounds__(kGradThreads) k_iota(int n, int* __restrict__ out) {
  const int i = (int)(blockIdx.x * (unsigned)kGradThreads + threadIdx.x);
  if (i < n) out[i] = i;
}

// start[p] / end[p] of point p's run in the sorted keys (both 0 for a point without observations: memset first)
__global__ void __launch_bounds__(kGradThreads) k_point_ranges(const int* __restrict__ key, int n, int* __restrict__ start,
                                                               int* __restrict__ end) {
  const int s = (int)(blockIdx.x * (unsigned)kGradThreads + threadIdx.x);
  if (s >= n) return;
  const int k = key[s];
  if (s == 0 || key[s - 1] != k) start[k] = s;
  if (s == n - 1 || key[s + 1] != k) end[k] = s + 1;
}

}  // namespace

struct svs_pose : svs::Handle {
  int max_obs = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int* d_pid = nullptr;
  double* d_obs = nullptr;
  double* d_xyz = nullptr;
  PoseCtl* d_ctl = nullptr;
  PoseCtl* h_ctl = nullptr;   // pinned
  // the last successful svs_calcFastMotionOnly / _device call, which svs_pose_grad differentiates: its inputs stay in
  // d_pid / d_obs / d_xyz, its pose in d_ctl->T
  bool have_problem = false;
  PoseArgs last{};
  int npoints = 0;
  bool sorted = false;          // order / start / end describe last's point ids
  // svs_pose_grad's buffers, allocated on its first call at the handle's capacity
  PoseGradCtl* d_gctl = nullptr;
  double* d_gout = nullptr;     // host outputs: dobs [max_obs][3] | dxyz [max_obs][3] | dcam [4]
  double* h_gout = nullptr;     // pinned: the same | a PoseGradCtl
  double* d_q = nullptr;        // [max_obs][3] point partials
  double* d_c = nullptr;        // [max_obs][4] camera partials
  int* d_sort = nullptr;        // keys | iota | order | start | end, max_obs each
  void* d_cub = nullptr;
  size_t cub_bytes = 0;
};

void svs::pose_capacity(const svs_pose* h, int* device, int* max_obs) { *device = h->device; *max_obs = h->max_obs; }

// after a successful array or device call: the problem svs_pose_grad differentiates
static void keep_problem(svs_pose* h, const PoseArgs& a, int npoints) {
  h->last = a;
  h->npoints = npoints;
  h->sorted = false;
  h->have_problem = true;
}

// src_pid (device input): the caller's obs.point_id, checked against npoints on the device on its way into h->d_pid
static int run(svs_pose* h, PoseArgs& a, const svs_cam* cam, const svs_pose_params* p, double T[7],
               svs_pose_stats* stats, const int* src_pid = nullptr, int npoints = 0) {
  a.f = cam->f; a.px = cam->px; a.py = cam->py; a.b = cam->b;
  a.robust = p->robust_kernel; a.num_iter = p->num_iter; a.kernel_param = p->kernel_param;
  a.initial_mu = p->initial_mu; a.tau = p->tau;
  memcpy(h->h_ctl->T, T, sizeof(double) * 7);
  h->h_ctl->bad_pid = 0;
  SVS_CK(h, cudaMemcpyAsync(h->d_ctl, h->h_ctl, offsetof(PoseCtl, bad_pid) + sizeof(int), cudaMemcpyHostToDevice, h->stream));
  if (src_pid) k_pose_ingest<<<(unsigned)((a.n + 255) / 256), 256, 0, h->stream>>>(src_pid, a.n, npoints, h->d_pid, h->d_ctl);
  SVS_CK(h, cudaEventRecord(h->ev0, h->stream));
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
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaEventRecord(h->ev1, h->stream));
  SVS_CK(h, cudaMemcpyAsync(h->h_ctl, h->d_ctl, sizeof(PoseCtl), cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  const PoseCtl& c = *h->h_ctl;
  if (c.bad_pid) { h->err = "obs.point_id outside point_list"; return SVS_ERR_INVALID; }
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
  svs_pose* h = new svs_pose();
  if (int rc = svs::open_handle(h, device)) {
    delete h;
    return rc;
  }
  h->max_obs = max_obs;
  const bool ok = cudaEventCreate(&h->ev0) == cudaSuccess && cudaEventCreate(&h->ev1) == cudaSuccess &&
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
  svs::begin_close(h);
  cudaFree(h->d_pid); cudaFree(h->d_obs); cudaFree(h->d_xyz); cudaFree(h->d_ctl);
  cudaFree(h->d_gctl); cudaFree(h->d_gout); cudaFree(h->d_q); cudaFree(h->d_c); cudaFree(h->d_sort); cudaFree(h->d_cub);
  if (h->h_gout) cudaFreeHost(h->h_gout);
  if (h->h_ctl) cudaFreeHost(h->h_ctl);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  delete h;
}

const char* svs_pose_last_error(const svs_pose* h) { return svs::last_error(h); }

int svs_calcFastMotionOnly(svs_pose* h, int n, const int* obs_point_id, const double* obs_uvu, int npoints,
                           const double* point_xyz, const svs_cam* cam, const svs_pose_params* params, double T_frame[7],
                           svs_pose_stats* stats) {
  svs::NvtxRange nvtx_("match");
  if (!h) return SVS_ERR_INVALID;
  h->have_problem = false;
  if (n <= 0 || !obs_point_id || !obs_uvu || npoints <= 0 || !point_xyz || !cam || !params || !T_frame)
    return SVS_ERR_INVALID;                       // the reference asserts obs_list.size() > 0
  if (n > h->max_obs || npoints > h->max_obs) { h->err = "more observations/points than the handle's capacity"; return SVS_ERR_INVALID; }
  for (int i = 0; i < n; ++i)
    if (obs_point_id[i] < 0 || obs_point_id[i] >= npoints) { h->err = "obs.point_id outside point_list"; return SVS_ERR_INVALID; }
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpyAsync(h->d_pid, obs_point_id, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaMemcpyAsync(h->d_obs, obs_uvu, sizeof(double) * 3 * (size_t)n, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaMemcpyAsync(h->d_xyz, point_xyz, sizeof(double) * 3 * (size_t)npoints, cudaMemcpyHostToDevice, h->stream));
  PoseArgs a;
  memset(&a, 0, sizeof a);
  a.pid = h->d_pid; a.obs = reinterpret_cast<const char*>(h->d_obs); a.xyz = reinterpret_cast<const char*>(h->d_xyz);
  a.obs_stride = a.xyz_stride = 3 * sizeof(double); a.n = n;
  const int rc = run(h, a, cam, params, T_frame, stats);
  if (rc == SVS_OK) keep_problem(h, a, npoints);
  return rc;
}

int svs_calcFastMotionOnly_device(svs_pose* h, int n, const int* obs_point_id, const double* obs_uvu, int npoints,
                                  const double* point_xyz, const svs_cam* cam, const svs_pose_params* params,
                                  double T_frame[7], svs_pose_stats* stats) {
  svs::NvtxRange nvtx_("match");
  if (!h) return SVS_ERR_INVALID;
  h->have_problem = false;
  if (n <= 0 || !obs_point_id || !obs_uvu || npoints <= 0 || !point_xyz || !cam || !params || !T_frame)
    return SVS_ERR_INVALID;
  if (n > h->max_obs || npoints > h->max_obs) { h->err = "more observations/points than the handle's capacity"; return SVS_ERR_INVALID; }
  for (const void* p : {(const void*)obs_point_id, (const void*)obs_uvu, (const void*)point_xyz})
    if (!svs::on_device(h->device, p)) {
      h->err = "svs_calcFastMotionOnly_device: an array is not device memory of the handle's device";
      return SVS_ERR_INVALID;
    }
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpyAsync(h->d_obs, obs_uvu, sizeof(double) * 3 * (size_t)n, cudaMemcpyDeviceToDevice, h->stream));
  SVS_CK(h, cudaMemcpyAsync(h->d_xyz, point_xyz, sizeof(double) * 3 * (size_t)npoints, cudaMemcpyDeviceToDevice, h->stream));
  PoseArgs a;
  memset(&a, 0, sizeof a);
  a.pid = h->d_pid; a.obs = reinterpret_cast<const char*>(h->d_obs); a.xyz = reinterpret_cast<const char*>(h->d_xyz);
  a.obs_stride = a.xyz_stride = 3 * sizeof(double); a.n = n;
  const int rc = run(h, a, cam, params, T_frame, stats, obs_point_id, npoints);   // obs_point_id is checked on its way in
  if (rc == SVS_OK) keep_problem(h, a, npoints);
  return rc;
}

int svs_pose_grad(svs_pose* h, double lambda, const double dL_dT[6], double* dL_dobs, double* dL_dxyz, double* dL_dcam,
                  int on_device, svs_pose_grad_stats* stats) {
  svs::NvtxRange nvtx_("poseGrad");
  if (!h) return SVS_ERR_INVALID;
  if (stats) memset(stats, 0, sizeof *stats);
  if (!h->have_problem) {
    h->err = "svs_pose_grad: no problem to differentiate (call svs_calcFastMotionOnly or _device first; a failed call "
             "and svs_calcFastMotionOnly_matched leave none)";
    return SVS_ERR_STATE;
  }
  if (!std::isfinite(lambda) || lambda < 0.) { h->err = "svs_pose_grad: lambda must be finite and >= 0"; return SVS_ERR_INVALID; }
  if (on_device)
    for (const void* p : {(const void*)dL_dT, (const void*)dL_dobs, (const void*)dL_dxyz, (const void*)dL_dcam})
      if (p && !svs::on_device(h->device, p)) {
        h->err = "svs_pose_grad: on_device = 1 but an array is not device memory of the handle's device";
        return SVS_ERR_INVALID;
      }
  cudaSetDevice(h->device);
  const int n = h->last.n, np = h->npoints, cap = h->max_obs;
  const size_t o_xyz = 3 * (size_t)cap, o_cam = 6 * (size_t)cap, o_ctl = o_cam + 4;   // offsets in d_gout / h_gout
  if (!h->d_gctl) {   // first gradient call on this handle (d_gctl last: it marks the set complete)
    if (!h->d_gout) SVS_CK(h, cudaMalloc(&h->d_gout, sizeof(double) * o_ctl));
    if (!h->h_gout) SVS_CK(h, cudaMallocHost(&h->h_gout, sizeof(double) * o_ctl + sizeof(PoseGradCtl)));
    if (!h->d_q) SVS_CK(h, cudaMalloc(&h->d_q, sizeof(double) * 3 * (size_t)cap));
    if (!h->d_c) SVS_CK(h, cudaMalloc(&h->d_c, sizeof(double) * 4 * (size_t)cap));
    if (!h->d_sort) SVS_CK(h, cudaMalloc(&h->d_sort, sizeof(int) * 5 * (size_t)cap));
    SVS_CK(h, cudaMalloc(&h->d_gctl, sizeof(PoseGradCtl)));
  }
  PoseGradCtl* h_gctl = reinterpret_cast<PoseGradCtl*>(h->h_gout + o_ctl);
  int* keys = h->d_sort; int* iota = keys + cap; int* order = iota + cap; int* start = order + cap; int* end = start + cap;
  const unsigned nblk = (unsigned)((n + kGradThreads - 1) / kGradThreads);
  // the stable sort of the observations by point, once per problem (only dL/dxyz needs it)
  if (dL_dxyz && !h->sorted) {
    int bits = 1;
    while (bits < 31 && (1 << bits) < np) ++bits;
    size_t need = 0;
    SVS_CK(h, cub::DeviceRadixSort::SortPairs(nullptr, need, h->last.pid, keys, iota, order, n, 0, bits, h->stream));
    if (need > h->cub_bytes) {
      SVS_CK(h, cudaFree(h->d_cub));
      h->d_cub = nullptr; h->cub_bytes = 0;
      SVS_CK(h, cudaMalloc(&h->d_cub, need));
      h->cub_bytes = need;
    }
    k_iota<<<nblk, kGradThreads, 0, h->stream>>>(n, iota);
    SVS_CK(h, cub::DeviceRadixSort::SortPairs(h->d_cub, need, h->last.pid, keys, iota, order, n, 0, bits, h->stream));
    SVS_CK(h, cudaMemsetAsync(start, 0, sizeof(int) * 2 * (size_t)cap, h->stream));   // start | end
    k_point_ranges<<<nblk, kGradThreads, 0, h->stream>>>(keys, n, start, end);
    SVS_CK(h, cudaGetLastError());
    h->sorted = true;
  }
  const double* g = dL_dT;
  double* go = dL_dobs; double* gx = dL_dxyz; double* gcam = dL_dcam;
  if (!on_device) {
    if (dL_dT) {
      memcpy(h_gctl->g, dL_dT, 6 * sizeof(double));
      SVS_CK(h, cudaMemcpyAsync(h->d_gctl->g, h_gctl->g, 6 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
      g = h->d_gctl->g;
    }
    go = go ? h->d_gout : nullptr;
    gx = gx ? h->d_gout + o_xyz : nullptr;
    gcam = gcam ? h->d_gout + o_cam : nullptr;
  }
  SVS_CK(h, cudaEventRecord(h->ev0, h->stream));
  const PoseArgs& a = h->last;
  if (n > kClusterMinObs) {   // the forward's launch shapes
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(kCl, 1, 1);
    cfg.blockDim = dim3(kClThreads, 1, 1);
    cfg.stream = h->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = kCl; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if (cudaLaunchKernelEx(&cfg, k_pose_grad_h<kClThreads, true>, a, (const PoseCtl*)h->d_ctl, g, lambda, h->d_gctl) !=
        cudaSuccess) {
      (void)cudaGetLastError();   // as in run(): the one-CTA shape
      k_pose_grad_h<kCtaThreads, false><<<1, kCtaThreads, 0, h->stream>>>(a, h->d_ctl, g, lambda, h->d_gctl);
    }
  } else {
    k_pose_grad_h<kCtaThreads, false><<<1, kCtaThreads, 0, h->stream>>>(a, h->d_ctl, g, lambda, h->d_gctl);
  }
  if (go || gx || gcam)
    k_pose_grad_obs<<<nblk, kGradThreads, 0, h->stream>>>(a, h->d_gctl, go, gx ? h->d_q : nullptr, gcam ? h->d_c : nullptr);
  if (gx)
    k_pose_grad_points<<<(unsigned)((np + kGradThreads - 1) / kGradThreads), kGradThreads, 0, h->stream>>>(
        order, start, end, h->d_q, np, h->d_gctl, gx);
  if (gcam) k_pose_grad_cam<<<1, kGradThreads, 0, h->stream>>>(h->d_c, n, h->d_gctl, gcam);
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaEventRecord(h->ev1, h->stream));
  if (!on_device) {
    if (go) SVS_CK(h, cudaMemcpyAsync(h->h_gout, go, sizeof(double) * 3 * (size_t)n, cudaMemcpyDeviceToHost, h->stream));
    if (gx) SVS_CK(h, cudaMemcpyAsync(h->h_gout + o_xyz, gx, sizeof(double) * 3 * (size_t)np, cudaMemcpyDeviceToHost, h->stream));
    if (gcam) SVS_CK(h, cudaMemcpyAsync(h->h_gout + o_cam, gcam, sizeof(double) * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  SVS_CK(h, cudaMemcpyAsync(h_gctl, h->d_gctl, sizeof(PoseGradCtl), cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  if (!on_device) {
    if (dL_dobs) memcpy(dL_dobs, h->h_gout, sizeof(double) * 3 * (size_t)n);
    if (dL_dxyz) memcpy(dL_dxyz, h->h_gout + o_xyz, sizeof(double) * 3 * (size_t)np);
    if (dL_dcam) memcpy(dL_dcam, h->h_gout + o_cam, sizeof(double) * 4);
  }
  if (stats) {
    stats->num_obs = n; stats->npoints = np;
    cudaEventElapsedTime(&stats->ms, h->ev0, h->ev1);
  }
  return h_gctl->fail ? 1 : 0;
}

int svs_calcFastMotionOnly_matched(svs_pose* h, svs_matcher* m, const svs_cam* cam, const svs_pose_params* params,
                                   double T_frame[7], svs_pose_stats* stats) {
  svs::NvtxRange nvtx_("match");
  if (!h) return SVS_ERR_INVALID;
  h->have_problem = false;   // svs_pose_grad does not differentiate through the matcher's buffers
  if (!m || !cam || !params || !T_frame) return SVS_ERR_INVALID;
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
