// dt.cu -- dense photometric SE3 tracker on sm_90a (ScaViSLAM GPU-path semantics).
//   scavislam/gpu/dense_tracking.cu:82-148   pointcloud_kernel / computePointCloud
//   scavislam/gpu/dense_tracking.cu:172-356  jacobianReduction_kernel + host-side final sum
//   scavislam/gpu/dense_tracking.cu:376-491  chi2_kernel + host-side final sum
//   scavislam/dense_tracking.cpp:62-216      DenseTracker::denseTrackingGpu / computeDensePointCloudGpu
//
// The reference launches a kernel, synchronises, copies per-block partials to the host and sums
// them there, twice per Levenberg trial.  Here one cooperative, persistent kernel per pyramid
// level runs the whole LM loop on the device: every trial is ONE fused pass over the pixels that
// yields chi2, J^T J and J^T r at the trial pose (an accepted trial's J^T J / J^T r are exactly
// what the reference's next jacobianReduction at the accepted pose would compute), a grid-wide
// deterministic reduction, and a 6x6 solve + SE3 exp by one thread.  HBM/L2-bound image work:
// ~20 B/pixel of compulsory reads (float4 cloud + previous intensity) plus 12 cached taps.
//
// Per-pixel arithmetic is IEEE single precision in the order the reference writes it (this
// translation unit is compiled with -fmad=false so that it matches the CPU oracle bit for bit);
// sums over pixels are accumulated in double (DESIGN.md, deviation D-DT1).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include "../../include/svs_b200.h"
#include "handle.cuh"
#include "se3_dev.cuh"
#include "svs_nvtx.hpp"

namespace cg = cooperative_groups;

namespace {

constexpr int kMaxLevels = 8;
constexpr int kThreads = 256;
constexpr int kAcc = 28;   // 21 Hessian + 6 gradient + chi2
constexpr int kPxBatch = 4;   // pixels a thread has in flight in the fused pass (accumulate_pass)

struct DtLevel {
  int w, h, stride, cloud_stride;
  float f, px, py;
  const float* prev;
  const float* cur;
  const float* dx;
  const float* dy;
  const float4* cloud;
};

struct DtCtl {
  double T[7];       // accepted pose (T_cur_from_actkey)
  double Teval[7];   // pose the next pass evaluates
  double H[21], b[6], chi2;
  double mu, nu;
  int trial, stop, iter, phase, done, passes;
  double chi2_level[kMaxLevels];
  int passes_level[kMaxLevels];
  // SVS_DT_TIMING: cycles per stage summed over the passes of a frame, per level [level][stage]: CTA 0's pose load,
  // pixel loop + CTA reduction, ticket, wait for the release; the last CTA's partial sums, decision + solve, release
  unsigned long long prof[kMaxLevels][8];
};

__device__ __forceinline__ float bilinear(const float* __restrict__ img, int stride, float u, float v, int exact) {
  const float x0 = floorf(u), y0 = floorf(v);
  float a = u - x0, b = v - y0;
  if (!exact) {   // texture-unit filtering: 8 fractional bits (dense_tracking.cu:285-287)
    a = floorf(a * 256.f + 0.5f) / 256.f;
    b = floorf(b * 256.f + 0.5f) / 256.f;
  }
  const int xi = (int)x0, yi = (int)y0;
  const float* p = img + (size_t)yi * stride + xi;
  const float t00 = __ldg(p), t10 = __ldg(p + 1), t01 = __ldg(p + stride), t11 = __ldg(p + stride + 1);
  return ((1.f - a) * (1.f - b)) * t00 + (a * (1.f - b)) * t10 + ((1.f - a) * b) * t01 + (a * b) * t11;
}

__device__ __forceinline__ void pose_to_m34(const double T[7], float m[12]) {
  double R[9];
  svs::quat_to_R(T, R);
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int r = 0; r < 3; ++r) m[c * 3 + r] = (float)R[r * 3 + c];
  m[9] = (float)T[4]; m[10] = (float)T[5]; m[11] = (float)T[6];
}

// one pixel of jacobianReduction_kernel / chi2_kernel (dense_tracking.cu:172-263, 376-453)
__device__ __forceinline__ bool pixel_terms(const DtLevel& L, const float m[12], int u, int v, int exact, bool want_jac,
                                            float& res, float jac[6]) {
  const float4 p = __ldg(L.cloud + (size_t)v * L.cloud_stride + u);
  if (!(p.w > 0)) return false;
  const float cx = p.x * m[0] + p.y * m[3] + p.z * m[6] + p.w * m[9];
  const float cy = p.x * m[1] + p.y * m[4] + p.z * m[7] + p.w * m[10];
  const float cz = p.x * m[2] + p.y * m[5] + p.z * m[8] + p.w * m[11];
  const float uc = L.f * cx / cz + L.px;
  const float vc = L.f * cy / cz + L.py;
  if (!(uc >= 1.f && vc >= 1.f && uc <= (float)(L.w - 2) && vc <= (float)(L.h - 2))) return false;
  const float ip = __ldg(L.prev + (size_t)v * L.stride + u);
  const float ic = bilinear(L.cur, L.stride, uc, vc, exact);
  res = ip - ic;
  if (want_jac) {
    float dx = 0.5f * bilinear(L.dx, L.stride, uc, vc, exact);
    float dy = 0.5f * bilinear(L.dy, L.stride, uc, vc, exact);
    const float z_sq = cz * cz;   // frameJacobian (dense_tracking.cu:65-80), literally
    dx *= L.f;
    dy *= L.f;
    jac[0] = (float)(-dx * (1. / cz));
    jac[1] = (float)(-dy * 1. / cz);
    jac[2] = (dx * cx / z_sq + dy * cy / z_sq);
    jac[3] = (dx * (cx * cy) / z_sq + dy * (1.f + cy * cy / z_sq));
    jac[4] = (-dx * (1.f + (cx * cx / z_sq)) - dy * (cx * cy) / z_sq);
    jac[5] = (dx * cy / cz - dy * cx / cz);
  }
  return true;
}

// per-thread accumulation over a grid-stride pixel range, then a fixed-order CTA reduction;
// partial[blockIdx][kAcc] (index 27 = chi2)
__device__ void accumulate_pass(const DtLevel& L, const double T[7], int exact, bool want_jac, double* __restrict__ partial,
                                double (*sred)[kAcc]) {
  float m[12];
  pose_to_m34(T, m);
  double acc[kAcc];
#pragma unroll
  for (int i = 0; i < kAcc; ++i) acc[i] = 0.;
  // kPxBatch pixels of the grid-stride sequence at a time, every load of the batch unconditional (a pixel that does
  // not contribute reads the taps of (1, 1) instead): the loads of the whole batch are in flight together, where the
  // one-pixel loop paid cloud -> taps -> next pixel's cloud -> ... in sequence.  Per-pixel arithmetic and the order
  // of the additions are those of pixel_terms / the one-pixel loop.
  const int npx = L.w * L.h;
  const int stride_px = gridDim.x * blockDim.x;
  if (npx <= 2 * stride_px) {   // coarse levels: one or two pixels per thread, nothing to batch
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < npx; idx += stride_px) {
      const int v = idx / L.w, u = idx - v * L.w;
      float res, jac[6];
      if (pixel_terms(L, m, u, v, exact, want_jac, res, jac)) {
        acc[27] += (double)(res * res);
        if (want_jac) {
          int i = 0;
#pragma unroll
          for (int r = 0; r < 6; ++r)
#pragma unroll
            for (int c = 0; c <= r; ++c) acc[i++] += (double)(jac[r] * jac[c]);
#pragma unroll
          for (int r = 0; r < 6; ++r) acc[21 + r] += (double)(jac[r] * res);
        }
      }
    }
  } else
  for (int idx0 = blockIdx.x * blockDim.x + threadIdx.x; idx0 < npx; idx0 += kPxBatch * stride_px) {
    int pu[kPxBatch], pv[kPxBatch];
    float4 pc[kPxBatch];
#pragma unroll
    for (int q = 0; q < kPxBatch; ++q) {
      const int idx = idx0 + q * stride_px;
      const bool in = idx < npx;
      const int ii = in ? idx : 0;
      pv[q] = ii / L.w; pu[q] = ii - pv[q] * L.w;
      pc[q] = __ldg(L.cloud + (size_t)pv[q] * L.cloud_stride + pu[q]);
      if (!in) pc[q].w = -1.f;
    }
    bool ok[kPxBatch];
    float cxq[kPxBatch], cyq[kPxBatch], czq[kPxBatch], ucq[kPxBatch], vcq[kPxBatch];
#pragma unroll
    for (int q = 0; q < kPxBatch; ++q) {
      const float4 p = pc[q];
      const float cx = p.x * m[0] + p.y * m[3] + p.z * m[6] + p.w * m[9];
      const float cy = p.x * m[1] + p.y * m[4] + p.z * m[7] + p.w * m[10];
      const float cz = p.x * m[2] + p.y * m[5] + p.z * m[8] + p.w * m[11];
      const float uc = L.f * cx / cz + L.px;
      const float vc = L.f * cy / cz + L.py;
      ok[q] = (p.w > 0) && (uc >= 1.f && vc >= 1.f && uc <= (float)(L.w - 2) && vc <= (float)(L.h - 2));
      cxq[q] = cx; cyq[q] = cy; czq[q] = cz;
      ucq[q] = ok[q] ? uc : 1.f; vcq[q] = ok[q] ? vc : 1.f;
    }
    float ipq[kPxBatch], icq[kPxBatch], dxq[kPxBatch], dyq[kPxBatch];
#pragma unroll
    for (int q = 0; q < kPxBatch; ++q) {
      ipq[q] = __ldg(L.prev + (size_t)pv[q] * L.stride + pu[q]);
      icq[q] = bilinear(L.cur, L.stride, ucq[q], vcq[q], exact);
      if (want_jac) {
        dxq[q] = bilinear(L.dx, L.stride, ucq[q], vcq[q], exact);
        dyq[q] = bilinear(L.dy, L.stride, ucq[q], vcq[q], exact);
      }
    }
#pragma unroll
    for (int q = 0; q < kPxBatch; ++q) {
      if (!ok[q]) continue;
      const float res = ipq[q] - icq[q];
      acc[27] += (double)(res * res);
      if (want_jac) {
        const float cx = cxq[q], cy = cyq[q], cz = czq[q];
        float jac[6];
        float dx = 0.5f * dxq[q];
        float dy = 0.5f * dyq[q];
        const float z_sq = cz * cz;   // frameJacobian (dense_tracking.cu:65-80), literally (as in pixel_terms)
        dx *= L.f;
        dy *= L.f;
        jac[0] = (float)(-dx * (1. / cz));
        jac[1] = (float)(-dy * 1. / cz);
        jac[2] = (dx * cx / z_sq + dy * cy / z_sq);
        jac[3] = (dx * (cx * cy) / z_sq + dy * (1.f + cy * cy / z_sq));
        jac[4] = (-dx * (1.f + (cx * cx / z_sq)) - dy * (cx * cy) / z_sq);
        jac[5] = (dx * cy / cz - dy * cx / cz);
        int i = 0;
#pragma unroll
        for (int r = 0; r < 6; ++r)
#pragma unroll
          for (int c = 0; c <= r; ++c) acc[i++] += (double)(jac[r] * jac[c]);
#pragma unroll
        for (int r = 0; r < 6; ++r) acc[21 + r] += (double)(jac[r] * res);
      }
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < kAcc; ++i) {
    double v = acc[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) sred[warp][i] = v;
  }
  __syncthreads();
  if (threadIdx.x < kAcc) {
    double s = 0;
    for (int w = 0; w < kThreads / 32; ++w) s += sred[w][threadIdx.x];
    partial[(size_t)blockIdx.x * kAcc + threadIdx.x] = s;
  }
  __syncthreads();   // (k_dt_track_level: thread 0 fences behind this barrier before it takes the ticket, which
                     //  publishes these stores to the CTA that sums the partials -- fences are cumulative)
}

// 1/a for the pivots of solve6: hardware approximation + two Newton steps (full double precision up to rounding).
// An IEEE double division is a ~25-instruction dependent sequence; the solve sits on the one-thread critical path of
// every LM pass (all other CTAs spin meanwhile), and the 21 divisions of the textbook LDL^T were most of it.
__device__ __forceinline__ double dt_inv(double a) {
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(a));
  double e = fma(-a, y, 1.0);
  y = fma(y, e, y);
  e = fma(-a, y, 1.0);
  return fma(y, e, y);
}

// (H + mu diag(H)) x = -b by LDL^T (H.ldlt().solve(-b), dense_tracking.cpp:127-135): in place on the packed lower
// triangle (H21[r (r + 1) / 2 + c]), six reciprocals and no division.  H21 / b6 may point to shared or global memory.
// kGlobal: the system lies in the control block in global memory, written by whichever CTA was last in an earlier pass:
// read it past L1 (ld.global.cg), which is not coherent between SMs.
template <bool kGlobal>
__device__ __forceinline__ void solve6(const double* __restrict__ H21, const double* __restrict__ b6, double mu, double x[6]) {
  double a[21], D[6], Di[6], bb[6];
#pragma unroll
  for (int i = 0; i < 21; ++i) a[i] = kGlobal ? __ldcg(H21 + i) : H21[i];
#pragma unroll
  for (int i = 0; i < 6; ++i) bb[i] = kGlobal ? __ldcg(b6 + i) : b6[i];
#pragma unroll
  for (int r = 0; r < 6; ++r) a[r * (r + 1) / 2 + r] += mu * a[r * (r + 1) / 2 + r];
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    double d = a[j * (j + 1) / 2 + j];
#pragma unroll
    for (int q = 0; q < j; ++q) d -= a[j * (j + 1) / 2 + q] * a[j * (j + 1) / 2 + q] * D[q];
    D[j] = d;
    Di[j] = d != 0. ? dt_inv(d) : 0.;
#pragma unroll
    for (int r = j + 1; r < 6; ++r) {
      double sv = a[r * (r + 1) / 2 + j];
#pragma unroll
      for (int q = 0; q < j; ++q) sv -= a[r * (r + 1) / 2 + q] * a[j * (j + 1) / 2 + q] * D[q];
      a[r * (r + 1) / 2 + j] = sv * Di[j];   // L[r][j]
    }
  }
  double y[6];
#pragma unroll
  for (int r = 0; r < 6; ++r) {
    double sv = -bb[r];
#pragma unroll
    for (int q = 0; q < r; ++q) sv -= a[r * (r + 1) / 2 + q] * y[q];
    y[r] = sv;
  }
#pragma unroll
  for (int r = 5; r >= 0; --r) {
    double sv = y[r] * Di[r];
#pragma unroll
    for (int q = r + 1; q < 6; ++q) sv -= a[q * (q + 1) / 2 + r] * x[q];
    x[r] = sv;
  }
}

// The Levenberg decision of one pass and the next trial pose (dense_tracking.cpp:105-178), run by thread 0 of the
// last CTA to arrive.  A function of its own (not inlined): its 27 + 14 doubles of state and the unrolled 6x6 solve
// would otherwise share the register allocation of the pixel loop.  Returns true when the level is finished.
__device__ __noinline__ bool decide_and_propose(DtCtl* c, const double* ssum, const double* Te, int pass, int level) {
  // The control block lives in global memory (the last CTA is a different one every pass).  What this decision needs
  // is fetched in ONE batch of independent loads; the block used to be read and written field by field, four or five
  // dependent L2 round trips per pass.
  double chi2 = 0, mu = 0, nu = 2, Tacc[7], b_old[6];
  int trial = 0, iter = 0, passes = 0;
  if (pass != 0) {
    chi2 = __ldcg(&c->chi2); mu = __ldcg(&c->mu); nu = __ldcg(&c->nu);
    trial = __ldcg(&c->trial); iter = __ldcg(&c->iter); passes = __ldcg(&c->passes);
#pragma unroll
    for (int k = 0; k < 7; ++k) Tacc[k] = __ldcg(&c->T[k]);
#pragma unroll
    for (int i = 0; i < 6; ++i) b_old[i] = __ldcg(&c->b[i]);
  }
  bool finished = false, new_system = false, new_pose = false;
  int stop = 0;
  if (pass == 0) {   // chi2 and (H, b) at the incoming pose (Te = ctl->T)
    passes = 1;
#pragma unroll
    for (int k = 0; k < 7; ++k) Tacc[k] = Te[k];
    chi2 = ssum[27];
    mu = (double)0.01f; nu = 2.; trial = 0; iter = 0;
    new_system = true;
    c->phase = 1;
  } else {
    passes += 1;
    const double chin = ssum[27];
    const double rho = chi2 - chin;
    if (rho > 0) {
#pragma unroll
      for (int k = 0; k < 7; ++k) Tacc[k] = Te[k];   // the evaluated pose is accepted
      new_pose = true;
      chi2 = chin;
      double nm = 0;
#pragma unroll
      for (int k = 0; k < 6; ++k) nm = fmax(nm, fabs(b_old[k]));   // b of the step just taken
      stop = nm <= 1e-10;   // norm_max(b) <= EPS
      const double u = 2 * rho - 1;
      mu *= fmax(1. / 3., 1 - u * u * u);
      nu = 2.;
      trial = 0;
      new_system = true;
      if (stop) finished = true;
      else { iter += 1; if (iter >= 15) finished = true; }
    } else {
      mu *= nu;
      nu *= 2.;
      trial += 1;
      if (trial == 2) { stop = 1; finished = true; }
    }
  }
  int done = 0;
  if (finished) {
    done = 1;
    c->chi2_level[level] = chi2;
    c->passes_level[level] = passes;
  } else {   // (H + mu diag H) x = -b, Teval = exp(x) T; the system of an accepted pass is still in shared memory
    double x[6], dT[7], Tev[7];
    if (new_system) solve6<false>(ssum, ssum + 21, mu, x);
    else solve6<true>(c->H, c->b, mu, x);
    svs::se3_exp(x, dT);
    svs::se3_mul(dT, Tacc, Tev);
#pragma unroll
    for (int k = 0; k < 7; ++k) c->Teval[k] = Tev[k];
  }
  // write back what changed (plain stores: nobody reads them before the next rendezvous)
  c->chi2 = chi2; c->mu = mu; c->nu = nu; c->trial = trial; c->iter = iter; c->passes = passes; c->stop = stop;
  c->done = done;
  if (new_pose) {
#pragma unroll
    for (int k = 0; k < 7; ++k) c->T[k] = Tacc[k];
  }
  if (new_system) {
#pragma unroll
    for (int i = 0; i < 21; ++i) c->H[i] = ssum[i];
#pragma unroll
    for (int i = 0; i < 6; ++i) c->b[i] = ssum[21 + i];
  }
  return done != 0;
}

// The LM loop of DenseTracker::denseTrackingGpu for one level (dense_tracking.cpp:90-178).
// One grid-wide rendezvous per pass: every CTA publishes its partial sums and takes a ticket; the LAST CTA to
// arrive sums the partials with all its threads in a fixed order (18 segments x 28 components, independent of
// which CTA happens to be last), takes the Levenberg decision, writes the next pose and bumps a generation
// counter the other CTAs spin on (all CTAs are co-resident: cooperative launch).
constexpr int kSeg = 18;
__global__ void __launch_bounds__(kThreads, 2)
k_dt_track_level(DtLevel L, DtCtl* ctl, double* partial, unsigned* sync, int exact, int level, int prof) {
  __shared__ double sred[kThreads / 32][kAcc];
  __shared__ double sseg[kSeg][kAcc];
  __shared__ double ssum[kAcc];
  __shared__ unsigned sGen;
  __shared__ int sLast;
  if (threadIdx.x == 0) sGen = *(volatile unsigned*)&sync[1];   // no CTA can bump it before every CTA has arrived once
  __syncthreads();
  unsigned gen = sGen & 0x7fffffffu;   // bit 31 = "level finished" of the previous launch
  for (int pass = 0;; ++pass) {
    double Te[7];
    const double* Tsrc = pass == 0 ? ctl->T : ctl->Teval;   // the first pass evaluates the incoming pose
    long long c0 = 0, c1 = 0, c2 = 0, c3 = 0;
    const bool stamp = prof && threadIdx.x == 0;
    if (stamp) c0 = clock64();
#pragma unroll
    for (int k = 0; k < 7; ++k) Te[k] = __ldcg(&Tsrc[k]);
    // (the comparison makes the stamp depend on the first loaded value, i.e. it is taken BEHIND the loads; it adds 0
    //  for any real pose, whose quaternion components lie in [-1, 1])
    if (stamp) { c1 = clock64() + (long long)(Te[0] == 123.456); }
    accumulate_pass(L, Te, exact, true, partial, sred);
    if (stamp) c2 = clock64();
    if (threadIdx.x == 0) {
      __threadfence();
      sLast = atomicAdd(&sync[0], 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (stamp) c3 = clock64();
    if (stamp && blockIdx.x == 0) {
      atomicAdd(&ctl->prof[level][0], (unsigned long long)(c1 - c0));
      atomicAdd(&ctl->prof[level][1], (unsigned long long)(c2 - c1));
      atomicAdd(&ctl->prof[level][2], (unsigned long long)(c3 - c2));
    }
    if (sLast) {
      __threadfence();
      if (threadIdx.x < 14 * kSeg) {
        // 18 segments x 14 lanes, each lane two components (one 16-byte load per partial), nine loads in flight:
        // 296 partials are two L2 round trips per lane.  Fixed order (b = seg, seg + 18, ...), independent of which
        // CTA happens to be the last.
        const int i2 = threadIdx.x % 14, seg = threadIdx.x / 14;
        double sx = 0, sy = 0;
        for (unsigned b0 = seg; b0 < gridDim.x; b0 += 9 * kSeg) {
          double2 v[9];
#pragma unroll
          for (int q = 0; q < 9; ++q) {
            const unsigned b = b0 + q * kSeg;
            v[q] = b < gridDim.x ? __ldcg(reinterpret_cast<const double2*>(partial + (size_t)b * kAcc) + i2) : make_double2(0., 0.);
          }
#pragma unroll
          for (int q = 0; q < 9; ++q) { sx += v[q].x; sy += v[q].y; }
        }
        sseg[seg][2 * i2] = sx;
        sseg[seg][2 * i2 + 1] = sy;
      }
      __syncthreads();
      if (threadIdx.x < kAcc) {
        double s = 0;
#pragma unroll
        for (int q = 0; q < kSeg; ++q) s += sseg[q][threadIdx.x];
        ssum[threadIdx.x] = s;
      }
      __syncthreads();
      long long c4 = 0;
      if (stamp) c4 = clock64();
      if (threadIdx.x == 0) {
        DtCtl* c = ctl;
        const bool level_done = decide_and_propose(c, ssum, Te, pass, level);
        long long c5 = 0;
        if (stamp) c5 = clock64();
        sync[0] = 0;
        __threadfence();
        // releases the other CTAs; bit 31 of the word they spin on says "level finished", so nobody needs another
        // L2 round trip for ctl->done (the next launch masks the bit off when it reads its starting generation)
        *(volatile unsigned*)&sync[1] = ((gen + 1u) & 0x7fffffffu) | (level_done ? 0x80000000u : 0u);
        if (stamp) {
          const long long c6 = clock64();
          atomicAdd(&c->prof[level][4], (unsigned long long)(c4 - c3));
          atomicAdd(&c->prof[level][5], (unsigned long long)(c5 - c4));
          atomicAdd(&c->prof[level][6], (unsigned long long)(c6 - c5));
        }
      }
    }
    if (threadIdx.x == 0) {
      unsigned g;
      while (((g = *(volatile unsigned*)&sync[1]) & 0x7fffffffu) == gen) {}
      __threadfence();
      sGen = g;
      if (stamp && blockIdx.x == 0) atomicAdd(&ctl->prof[level][3], (unsigned long long)(clock64() - c3));
    }
    __syncthreads();
    gen = (gen + 1u) & 0x7fffffffu;
    if (sGen & 0x80000000u) break;   // (sGen is next written behind the barriers of the next pass)
  }
}

// GpuTracker::chi2 / jacobianReduction as stand-alone launches (parity hooks)
__global__ void __launch_bounds__(kThreads)
k_dt_pass(DtLevel L, const double* T, double* partial, int exact, int want_jac) {
  __shared__ double sred[kThreads / 32][kAcc];
  double Te[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) Te[k] = T[k];
  accumulate_pass(L, Te, exact, want_jac != 0, partial, sred);
}

// residualImage_kernel (dense_tracking.cu:494-541): the per-pixel visualisation of the photometric residual at the
// final pose of a level -- grey max(0, 1 - 50 r^2) where the pixel contributes, red where it projects outside the
// frame, green where it has no depth; packed float4 rows (w * h)
__global__ void k_dt_residual_image(DtLevel L, const double* __restrict__ T, int exact, float4* __restrict__ out) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  const int v = blockIdx.y * blockDim.y + threadIdx.y;
  if (u >= L.w || v >= L.h) return;
  double Te[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) Te[k] = T[k];
  float m[12];
  pose_to_m34(Te, m);
  float4 o;
  const float4 p = __ldg(L.cloud + (size_t)v * L.cloud_stride + u);
  if (p.w > 0) {
    float res, jac[6];
    if (pixel_terms(L, m, u, v, exact, false, res, jac)) {
      const float g = fmaxf(0.f, 1 - 50.f * res * res);
      o = make_float4(g, g, g, 1.f);
    } else {
      o = make_float4(1.f, 0.f, 0.f, 1.f);
    }
  } else {
    o = make_float4(0.f, 1.f, 0.f, 1.f);
  }
  out[(size_t)v * L.w + u] = o;
}

// pointcloud_kernel (dense_tracking.cu:82-122)
struct M4 { float m[16]; };
__global__ void k_dt_pointcloud(M4 TQ, const float* __restrict__ disp, int width, int height, int stride_in, int stride_out,
                                int factor, float4* __restrict__ cloud) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  const int v = blockIdx.y * blockDim.y + threadIdx.y;
  if (u >= width || v >= height) return;
  const int idx_in = v * stride_in + u * factor;   // row not scaled by factor, as in the reference (SURVEY B13)
  const float d = disp[idx_in] * factor;
  float4 pt;
  if (d <= 0) {
    pt = make_float4(0.f, 0.f, 0.f, -1.f);
  } else {
    const float uvd[4] = {(float)u, (float)v, d, 1.f};
    float p[4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
      p[r] = uvd[0] * TQ.m[r] + uvd[1] * TQ.m[4 + r] + uvd[2] * TQ.m[8 + r] + uvd[3] * TQ.m[12 + r];
    pt = make_float4(p[0] / p[3], p[1] / p[3], p[2] / p[3], 1.f);
  }
  cloud[(size_t)v * stride_out + u] = pt;
}

}  // namespace

struct svs_dt : svs::Handle {
  int nlevels = 0, w0 = 0, h0 = 0, flags = 0;
  DtLevel lv[kMaxLevels];
  float* img[kMaxLevels][4] = {};   // prev cur dx dy
  float4* cloud[kMaxLevels] = {};
  float* disp = nullptr;
  int disp_stride = 0, disp_w = 0, disp_h = 0;
  DtCtl* d_ctl = nullptr;
  DtCtl* h_ctl = nullptr;
  double* d_partial = nullptr;
  double* d_T = nullptr;
  unsigned* d_sync = nullptr;   // ticket, generation of k_dt_track_level
  float4* d_res = nullptr;      // residual image of the largest level (made on the first svs_dt_residual_image)
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int max_blocks = 0, track_blocks = 0;
  float* stage = nullptr;   // pinned staging for image uploads
  size_t stage_floats = 0;
};

extern "C" {

int svs_dt_create(int device, int w0, int h0, int nlevels, int flags, svs_dt** out) {
  if (!out || w0 <= 0 || h0 <= 0 || nlevels <= 0 || nlevels > kMaxLevels) return SVS_ERR_INVALID;
  *out = nullptr;
  svs_dt* h = new svs_dt();
  if (int rc = svs::open_handle(h, device)) {
    delete h;
    return rc;
  }
  h->nlevels = nlevels; h->w0 = w0; h->h0 = h0; h->flags = flags;
  bool ok = true;
  for (int l = 0; ok && l < nlevels; ++l) {
    const int w = w0 >> l, hh = h0 >> l;
    DtLevel& L = h->lv[l];
    L.w = w; L.h = hh; L.stride = ((w + 63) / 64) * 64; L.cloud_stride = L.stride;
    L.f = 1.f; L.px = 0.f; L.py = 0.f;
    for (int k = 0; ok && k < 4; ++k) {
      ok = cudaMalloc(&h->img[l][k], sizeof(float) * (size_t)L.stride * hh) == cudaSuccess &&
           cudaMemset(h->img[l][k], 0, sizeof(float) * (size_t)L.stride * hh) == cudaSuccess;
    }
    ok = ok && cudaMalloc(&h->cloud[l], sizeof(float4) * (size_t)L.cloud_stride * hh) == cudaSuccess &&
         cudaMemset(h->cloud[l], 0, sizeof(float4) * (size_t)L.cloud_stride * hh) == cudaSuccess;
    L.prev = h->img[l][0]; L.cur = h->img[l][1]; L.dx = h->img[l][2]; L.dy = h->img[l][3]; L.cloud = h->cloud[l];
  }
  h->disp_stride = ((w0 + 63) / 64) * 64;
  ok = ok && cudaMalloc(&h->disp, sizeof(float) * (size_t)h->disp_stride * h0) == cudaSuccess;
  int per_sm = 0, sms = 0;
  if (ok) {
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_dt_track_level, kThreads, 0);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    h->max_blocks = std::max(1, per_sm * sms);
    // the tracker's passes are latency-bound (rendezvous + 6x6 solve per pass): two CTAs per SM keep the
    // final sum short and still cover a 640x480 level with 4 pixels per thread
    h->track_blocks = std::max(1, std::min(per_sm, 2) * sms);
  }
  const int part_blocks = std::max(h->max_blocks, (w0 * h0 + kThreads - 1) / kThreads);
  ok = ok && cudaMalloc(&h->d_ctl, sizeof(DtCtl)) == cudaSuccess && cudaMemset(h->d_ctl, 0, sizeof(DtCtl)) == cudaSuccess &&
       cudaMalloc(&h->d_partial, sizeof(double) * kAcc * (size_t)part_blocks) == cudaSuccess &&
       cudaMalloc(&h->d_T, sizeof(double) * 8) == cudaSuccess &&
       cudaMalloc(&h->d_sync, sizeof(unsigned) * 2) == cudaSuccess && cudaMemset(h->d_sync, 0, sizeof(unsigned) * 2) == cudaSuccess &&
       cudaEventCreate(&h->ev0) == cudaSuccess && cudaEventCreate(&h->ev1) == cudaSuccess &&
       cudaMallocHost(&h->h_ctl, sizeof(DtCtl)) == cudaSuccess;
  h->stage_floats = (size_t)h->disp_stride * h0 * 4;
  ok = ok && cudaMallocHost(&h->stage, sizeof(float) * h->stage_floats) == cudaSuccess;
  if (!ok) {
    svs_dt_destroy(h);
    return SVS_ERR_CUDA;
  }
  *out = h;
  return SVS_OK;
}

void svs_dt_destroy(svs_dt* h) {
  if (!h) return;
  svs::begin_close(h);
  for (int l = 0; l < kMaxLevels; ++l) {
    for (int k = 0; k < 4; ++k) cudaFree(h->img[l][k]);
    cudaFree(h->cloud[l]);
  }
  cudaFree(h->disp); cudaFree(h->d_ctl); cudaFree(h->d_partial); cudaFree(h->d_T); cudaFree(h->d_sync); cudaFree(h->d_res);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->h_ctl) cudaFreeHost(h->h_ctl);
  if (h->stage) cudaFreeHost(h->stage);
  delete h;
}

const char* svs_dt_last_error(const svs_dt* h) { return svs::last_error(h); }

int svs_dt_set_intrinsics(svs_dt* h, int level, float focal_length, float px, float py) {
  if (!h || level < 0 || level >= h->nlevels) return SVS_ERR_INVALID;
  h->lv[level].f = focal_length; h->lv[level].px = px; h->lv[level].py = py;
  return SVS_OK;
}

static int upload_plane(svs_dt* h, float* dst, int dst_stride, const float* src, int src_stride, int w, int hgt) {
  SVS_CK(h, cudaMemcpy2DAsync(dst, sizeof(float) * dst_stride, src, sizeof(float) * src_stride, sizeof(float) * w, hgt,
                              cudaMemcpyHostToDevice, h->stream));
  return SVS_OK;
}

int svs_dt_set_images(svs_dt* h, int level, const float* prev, const float* cur, const float* dx, const float* dy,
                      int stride_floats) {
  if (!h || level < 0 || level >= h->nlevels || stride_floats < h->lv[level].w) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  const DtLevel& L = h->lv[level];
  const float* src[4] = {prev, cur, dx, dy};
  for (int k = 0; k < 4; ++k)
    if (src[k]) {
      int rc = upload_plane(h, h->img[level][k], L.stride, src[k], stride_floats, L.w, L.h);
      if (rc) return rc;
    }
  return SVS_OK;
}

// same planes already on the device (e.g. svs_prep_level pointers): device-to-device copies
int svs_dt_set_images_device(svs_dt* h, int level, const float* prev, const float* cur, const float* dx, const float* dy,
                             int stride_floats) {
  if (!h || level < 0 || level >= h->nlevels || stride_floats < h->lv[level].w) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  const DtLevel& L = h->lv[level];
  const float* src[4] = {prev, cur, dx, dy};
  for (int k = 0; k < 4; ++k)
    if (src[k])
      SVS_CK(h, cudaMemcpy2DAsync(h->img[level][k], sizeof(float) * L.stride, src[k], sizeof(float) * stride_floats,
                                  sizeof(float) * L.w, L.h, cudaMemcpyDeviceToDevice, h->stream));
  return SVS_OK;
}

// the current images become the previous ones (frame hand-over of FrameData::nextFrame)
int svs_dt_swap_prev_cur(svs_dt* h) {
  if (!h) return SVS_ERR_INVALID;
  for (int l = 0; l < h->nlevels; ++l) {
    std::swap(h->img[l][0], h->img[l][1]);
    h->lv[l].prev = h->img[l][0]; h->lv[l].cur = h->img[l][1];
  }
  return SVS_OK;
}

int svs_dt_set_disparity(svs_dt* h, const float* disp, int stride_floats, int w, int hgt) {
  if (!h || !disp || w <= 0 || hgt <= 0 || w > h->w0 || hgt > h->h0 || stride_floats < w) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  h->disp_w = w; h->disp_h = hgt;
  return upload_plane(h, h->disp, h->disp_stride, disp, stride_floats, w, hgt);
}

// the same map already on this device (svs_stereo_disparity): a device-to-device copy; on return the source may change
int svs_dt_set_disparity_device(svs_dt* h, const float* d_disp, int stride_floats, int w, int hgt) {
  if (!h || !d_disp || w <= 0 || hgt <= 0 || w > h->w0 || hgt > h->h0 || stride_floats < w) return SVS_ERR_INVALID;
  if (!svs::on_device(h->device, d_disp)) return svs::fail(h, SVS_ERR_INVALID, "svs_dt_set_disparity_device: not device memory of this handle's device");
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpy2DAsync(h->disp, sizeof(float) * h->disp_stride, d_disp, sizeof(float) * stride_floats, sizeof(float) * w, hgt,
                              cudaMemcpyDeviceToDevice, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  h->disp_w = w; h->disp_h = hgt;
  return SVS_OK;
}

int svs_dt_set_point_cloud(svs_dt* h, int level, const float* cloud_xyzw) {
  if (!h || level < 0 || level >= h->nlevels || !cloud_xyzw) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  const DtLevel& L = h->lv[level];
  SVS_CK(h, cudaMemcpy2DAsync(h->cloud[level], sizeof(float4) * L.cloud_stride, cloud_xyzw, sizeof(float4) * L.w,
                              sizeof(float4) * L.w, L.h, cudaMemcpyHostToDevice, h->stream));
  return SVS_OK;
}

int svs_dt_get_point_cloud(svs_dt* h, int level, float* cloud_xyzw) {
  if (!h || level < 0 || level >= h->nlevels || !cloud_xyzw) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  const DtLevel& L = h->lv[level];
  SVS_CK(h, cudaMemcpy2DAsync(cloud_xyzw, sizeof(float4) * L.w, h->cloud[level], sizeof(float4) * L.cloud_stride,
                              sizeof(float4) * L.w, L.h, cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  return SVS_OK;
}

// DenseTracker::computeDensePointCloudGpu (dense_tracking.cpp:195-216): per level TQ = T^-1 Q(level camera)
int svs_dt_compute_point_cloud(svs_dt* h, const double T_cur_from_actkey[7], const svs_cam* cams) {
  svs::NvtxRange nvtx_("dense point cloud");
  if (!h || !T_cur_from_actkey || !cams) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  // T^-1 in double
  const double* T = T_cur_from_actkey;
  const double qi[4] = {-T[0], -T[1], -T[2], T[3]};
  double R[9];
  {
    const double x = qi[0], y = qi[1], z = qi[2], w = qi[3];
    R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w); R[2] = 2 * (x * z + y * w);
    R[3] = 2 * (x * y + z * w); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
    R[6] = 2 * (x * z - y * w); R[7] = 2 * (y * z + x * w); R[8] = 1 - 2 * (x * x + y * y);
  }
  double ti[3];
  for (int r = 0; r < 3; ++r) ti[r] = -(R[r * 3] * T[4] + R[r * 3 + 1] * T[5] + R[r * 3 + 2] * T[6]);
  for (int l = 0; l < h->nlevels; ++l) {
    const svs_cam& c = cams[l];
    double M[16] = {R[0], R[1], R[2], ti[0], R[3], R[4], R[5], ti[1], R[6], R[7], R[8], ti[2], 0, 0, 0, 1};
    const double Q[16] = {1, 0, 0, -c.px, 0, 1, 0, -c.py, 0, 0, 0, c.f, 0, 0, 1. / c.b, 0};   // stereo_camera.cpp:24-34
    M4 TQ;
    for (int r = 0; r < 4; ++r)
      for (int cc = 0; cc < 4; ++cc) {
        double s = 0;
        for (int k = 0; k < 4; ++k) s += M[r * 4 + k] * Q[k * 4 + cc];
        TQ.m[cc * 4 + r] = (float)s;
      }
    const DtLevel& L = h->lv[l];
    const dim3 blk(32, 8), grd((L.w + 31) / 32, (L.h + 7) / 8);
    k_dt_pointcloud<<<grd, blk, 0, h->stream>>>(TQ, h->disp, L.w, L.h, h->disp_stride, L.cloud_stride, 1 << l, h->cloud[l]);
  }
  SVS_CK(h, cudaGetLastError());
  return SVS_OK;
}

static int run_pass(svs_dt* h, int level, const double T[7], int want_jac, double sums[kAcc]) {
  if (!h || level < 0 || level >= h->nlevels || !T) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  const DtLevel& L = h->lv[level];
  const int blocks = std::min(h->max_blocks, std::max(1, (L.w * L.h + kThreads - 1) / kThreads));
  SVS_CK(h, cudaMemcpyAsync(h->d_T, T, sizeof(double) * 7, cudaMemcpyHostToDevice, h->stream));
  k_dt_pass<<<blocks, kThreads, 0, h->stream>>>(L, h->d_T, h->d_partial, (h->flags & SVS_DT_EXACT_BILINEAR) ? 1 : 0, want_jac);
  std::vector<double> part((size_t)blocks * kAcc);
  SVS_CK(h, cudaMemcpyAsync(part.data(), h->d_partial, sizeof(double) * part.size(), cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  SVS_CK(h, cudaGetLastError());
  for (int i = 0; i < kAcc; ++i) {
    double s = 0;
    for (int b = 0; b < blocks; ++b) s += part[(size_t)b * kAcc + i];
    sums[i] = s;
  }
  return SVS_OK;
}

int svs_dt_chi2(svs_dt* h, int level, const double T[7], double* chi2) {
  double s[kAcc];
  int rc = run_pass(h, level, T, 0, s);
  if (rc) return rc;
  *chi2 = s[27];
  return SVS_OK;
}

int svs_dt_jacobian_reduction(svs_dt* h, int level, const double T[7], double H21[21], double b6[6], double* chi2) {
  double s[kAcc];
  int rc = run_pass(h, level, T, 1, s);
  if (rc) return rc;
  memcpy(H21, s, sizeof(double) * 21);
  memcpy(b6, s + 21, sizeof(double) * 6);
  if (chi2) *chi2 = s[27];
  return SVS_OK;
}

int svs_dt_residual_image(svs_dt* h, int level, const double T[7], float* res_rgba) {
  if (!h || level < 0 || level >= h->nlevels || !T || !res_rgba) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  const DtLevel& L = h->lv[level];
  if (!h->d_res) SVS_CK(h, cudaMalloc(&h->d_res, sizeof(float4) * (size_t)h->w0 * h->h0));
  SVS_CK(h, cudaMemcpyAsync(h->d_T, T, sizeof(double) * 7, cudaMemcpyHostToDevice, h->stream));
  const dim3 block(32, 8), grid((L.w + 31) / 32, (L.h + 7) / 8);
  k_dt_residual_image<<<grid, block, 0, h->stream>>>(L, h->d_T, (h->flags & SVS_DT_EXACT_BILINEAR) ? 1 : 0, h->d_res);
  SVS_CK(h, cudaMemcpyAsync(res_rgba, h->d_res, sizeof(float4) * (size_t)L.w * L.h, cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  SVS_CK(h, cudaGetLastError());
  return SVS_OK;
}

int svs_dt_track(svs_dt* h, double T[7], svs_dt_stats* st) {
  svs::NvtxRange nvtx_("dense tracking");
  if (!h || !T) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpyAsync(h->d_ctl, T, sizeof(double) * 7, cudaMemcpyHostToDevice, h->stream));   // DtCtl::T is first
  cudaEvent_t e0 = h->ev0, e1 = h->ev1;   // created once with the handle: nothing is allocated per frame
  cudaEventRecord(e0, h->stream);
  int exact = (h->flags & SVS_DT_EXACT_BILINEAR) ? 1 : 0;
  for (int l = h->nlevels - 1; l >= 0; --l) {
    DtLevel L = h->lv[l];
    int blocks = std::min(h->track_blocks, std::max(1, (L.w * L.h + kThreads - 1) / kThreads));
    DtCtl* ctl = h->d_ctl;
    double* part = h->d_partial;
    unsigned* sync = h->d_sync;
    int level = l;
    static const int prof_on = getenv("SVS_DT_TIMING") ? 1 : 0;
    int prof = prof_on;
    void* args[] = {&L, &ctl, &part, &sync, &exact, &level, &prof};
    SVS_CK(h, cudaLaunchCooperativeKernel((void*)k_dt_track_level, dim3(blocks), dim3(kThreads), args, 0, h->stream));
  }
  cudaEventRecord(e1, h->stream);
  SVS_CK(h, cudaMemcpyAsync(h->h_ctl, h->d_ctl, sizeof(DtCtl), cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  SVS_CK(h, cudaGetLastError());
  memcpy(T, h->h_ctl->T, sizeof(double) * 7);
  if (getenv("SVS_DT_TIMING")) {   // cumulative over the handle's frames (the control block is only zeroed at creation)
    static const char* names[7] = {"pose load", "pixels+reduce", "ticket", "wait(release)", "last: partial sums", "last: decide+solve", "last: release"};
    for (int l = h->nlevels - 1; l >= 0; --l) {
      fprintf(stderr, "svs_dt level %d passes(last frame) %d cycles:", l, h->h_ctl->passes_level[l]);
      for (int q = 0; q < 7; ++q) fprintf(stderr, " %s=%llu", names[q], h->h_ctl->prof[l][q]);
      fprintf(stderr, "\n");
    }
  }
  if (st) {
    memset(st, 0, sizeof *st);
    cudaEventElapsedTime(&st->ms_total, e0, e1);
    for (int l = 0; l < h->nlevels && l < SVS_DT_MAX_LEVELS; ++l) {
      st->chi2[l] = h->h_ctl->chi2_level[l];
      st->passes[l] = h->h_ctl->passes_level[l];
      st->launches += 1;
    }
  }
  return SVS_OK;
}

}  // extern "C"
