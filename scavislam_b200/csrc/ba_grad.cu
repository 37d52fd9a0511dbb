// ba_grad.cu -- the adjoint of an optimised window (svs_ba_observation_grad): dL/d(observations, weights) from the
// upstream gradient g = (dL/d delta_p, dL/d psi_l) by one solve (H + lambda I) v = g.
//
// With H = [[A, B], [B^T, C]] over (poses, landmarks), Hpl_a = BaDev::W of slot a and D = (Hll + lambda I)^-1 from
// BaDev::Dbl, as the build left them:
//   k_grad_rhs    bp = g_p (0 for a fixed pose), bc = sum_l sum_a Hpl_a D g_l; k_solve then gives x = v_p = S^-1 (bp - bc)
//   k_grad_edges  v_l = D (g_l - sum_a Hpl_a^T v_pa), then per edge e of l, with J_e = de_e/dx unscaled at the accepted
//                 state, dL/dz_e = -rho' Omega_e (J_e v) and dL/domega_e = -rho' e_e (.) (J_e v), written at edge_src[e].
// Fixed poses have Hpl = 0 and x = 0 and add exactly nothing.  The self edge (pose == anchor) has J_pose = -J_anchor, so
// only its psi block acts on v.  Each caller edge is written by exactly one lane and every sum runs in a fixed order.
// svs_ba_window_grad adds, from the same v:
//   k_grad_edges<., true>  also the camera term per landmark, sum over its edges of (de_e/dcam)^T dL/dz_e (e is linear in
//                          z, so dL/dcam is the contraction of dL/dz), one partial [4] per landmark
//   k_grad_cam             the L partials summed in a fixed order by one CTA: no atomics, the same bits on every run
//   k_grad_constraints     one thread per pose-pose constraint: w_c = J_i v_i + J_j v_j, dL/dLambda_c, dL/d delta_c
#include "ba_dev.cuh"
#include "ba_kernels.cuh"

namespace svs {

namespace {

constexpr int kGradThreads = 256;
constexpr int kShortTrack = 8;   // slots of a track a group of kShortLanes lanes takes; longer tracks get a warp
constexpr int kShortLanes = 8;

// One thread per landmark: u = D g_l, then Hpl_a u into bc of every slot's pose; threads past L fill bp.
__global__ void __launch_bounds__(kGradThreads)
k_grad_rhs(BaDev d, const double* __restrict__ g_pose, const double* __restrict__ g_psi, double lambda) {
  const int i = (int)(blockIdx.x * (unsigned)kGradThreads + threadIdx.x);
  if (i >= d.L) {
    const int q = i - d.L;
    if (q < 6 * d.P) d.bp[q] = (g_pose && !__ldg(d.fixed + q / 6)) ? __ldg(g_pose + q) : 0.;
    return;
  }
  const int li = i;
  if (!g_psi || __ldg(d.lm_eptr + li + 1) == __ldg(d.lm_eptr + li)) return;   // no edges: not a variable
  const double* gl = g_psi + 3 * (size_t)__ldg(d.lm_user + li);
  const double g0 = __ldg(gl), g1 = __ldg(gl + 1), g2 = __ldg(gl + 2);
  double D[9];
  inv3_sym_lambda(d.Dbl + 12 * (size_t)li, lambda, D);
  const double u[3] = {D[0] * g0 + D[1] * g1 + D[2] * g2, D[3] * g0 + D[4] * g1 + D[5] * g2,
                       D[6] * g0 + D[7] * g1 + D[8] * g2};
  const int s0 = __ldg(d.lm_sptr + li), K = __ldg(d.lm_sptr + li + 1) - s0;
  const int e0 = __ldg(d.lm_eptr + li), off = __ldg(d.lm_self + li) ? 0 : 1, ia = __ldg(d.lm_anchor + li);
  const size_t ns = (size_t)d.nslots;
  for (int a = 0; a < K; ++a) {
    const int p = a == 0 ? ia : __ldg(d.e_pose + e0 + a - off);
    if (d.fixed[p]) continue;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
      const double* w = d.W + (size_t)(3 * r) * ns + s0 + a;
      atomicAdd(d.bc + 6 * p + r, __ldg(w) * u[0] + __ldg(w + ns) * u[1] + __ldg(w + 2 * ns) * u[2]);
    }
  }
}

// One group of LANES lanes per landmark of `list` (nullptr: landmark idx) whose slot count falls on this instance's
// side of kShortTrack.  Lane `sub` takes the slots and then the edges sub, sub + LANES, ...; the slot sums are reduced
// over the group by a butterfly, which leaves the same bits on every lane.  kCam: the group's camera sums are reduced
// by the same butterfly and lane 0 writes cam_part[li] (0 for a landmark without edges).
template <int LANES, bool kCam>
__global__ void __launch_bounds__(kGradThreads)
k_grad_edges(BaDev d, const int* __restrict__ list, int n, const double* __restrict__ g_psi, double lambda, int robust,
             double delta, double* __restrict__ dobs, double* __restrict__ dinfo, double* __restrict__ cam_part) {
  const int lane = threadIdx.x & 31, sub = lane & (LANES - 1);
  const int idx = (int)((blockIdx.x * (unsigned)kGradThreads + threadIdx.x) / LANES);
  if (idx >= n) return;   // whole groups leave together
  const int li = list ? __ldg(list + idx) : idx;
  const int s0 = __ldg(d.lm_sptr + li), K = __ldg(d.lm_sptr + li + 1) - s0;
  if ((K > kShortTrack) != (LANES == 32)) return;   // the other instance's landmark
  const unsigned gmask = LANES == 32 ? 0xffffffffu : ((1u << LANES) - 1u) << (lane & ~(LANES - 1));
  const int e0 = __ldg(d.lm_eptr + li), k = __ldg(d.lm_eptr + li + 1) - e0;
  if (k == 0) {
    if (kCam && sub == 0)
#pragma unroll
      for (int q = 0; q < 4; ++q) cam_part[4 * (size_t)li + q] = 0.;
    return;
  }
  const bool failed = d.ctl->chol_fail;
  const int off = __ldg(d.lm_self + li) ? 0 : 1, ia = __ldg(d.lm_anchor + li);
  const size_t ns = (size_t)d.nslots;
  const double* __restrict__ x = d.x;
  // t = sum_a Hpl_a^T v_pa
  double t[3] = {0., 0., 0.};
  for (int a = sub; a < K && !failed; a += LANES) {
    const int p = a == 0 ? ia : __ldg(d.e_pose + e0 + a - off);
#pragma unroll
    for (int r = 0; r < 6; ++r) {
      const double v = x[6 * p + r];
#pragma unroll
      for (int i = 0; i < 3; ++i) t[i] = fma(__ldg(d.W + (size_t)(3 * r + i) * ns + s0 + a), v, t[i]);
    }
  }
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int s = LANES / 2; s > 0; s >>= 1) t[i] += __shfl_xor_sync(gmask, t[i], s);
  double vl[3] = {0., 0., 0.};
  if (!failed) {
    double D[9];
    inv3_sym_lambda(d.Dbl + 12 * (size_t)li, lambda, D);
    double r[3] = {-t[0], -t[1], -t[2]};
    if (g_psi) {
      const double* gl = g_psi + 3 * (size_t)__ldg(d.lm_user + li);
      r[0] += __ldg(gl); r[1] += __ldg(gl + 1); r[2] += __ldg(gl + 2);
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) vl[i] = D[3 * i] * r[0] + D[3 * i + 1] * r[1] + D[3 * i + 2] * r[2];
  }
  const int cur = d.ctl->cur;
  const double* __restrict__ Rt = d.Rt[cur];
  const double* __restrict__ psi = d.psi[cur] + 3 * (size_t)li;
  double Ra[9], ta[3];
  load12(Rt, ia, Ra, ta);
  const double ipz = 1. / __ldg(psi + 2);
  const double xa[3] = {__ldg(psi) * ipz, __ldg(psi + 1) * ipz, ipz};   // invert_depth (maths_utils.h:66-69)
  double va[6];
#pragma unroll
  for (int r = 0; r < 6; ++r) va[r] = x[6 * ia + r];
  double gc[4] = {0., 0., 0., 0.};   // kCam: dL/d(f, px, py, b) of this lane's edges
  for (int i = sub; i < k; i += LANES) {
    const int e = e0 + i, src = __ldg(d.edge_src + e);
    if (src < 0) continue;   // zero-weight padding edge
    const double om[3] = {__ldg(d.e_w + e), __ldg(d.e_w + (size_t)d.E + e), __ldg(d.e_w + 2 * (size_t)d.E + e)};
    double go[3] = {0., 0., 0.}, gw[3] = {0., 0., 0.};
    if (!failed && (om[0] != 0. || om[1] != 0. || om[2] != 0.)) {   // the build never evaluates a zero-weight edge
      const int ip = __ldg(d.e_pose + e);
      const double obs[3] = {__ldg(d.e_obs + e), __ldg(d.e_obs + (size_t)d.E + e), __ldg(d.e_obs + 2 * (size_t)d.E + e)};
      double Rc[9], tc[3], R[9], tr[3], y[3], er[3];
      load12(Rt, ip, Rc, tc);
      rel_pose(Rc, tc, Ra, ta, R, tr);
      mat3_vec(R, xa, y);
      y[0] += tr[0]; y[1] += tr[1]; y[2] += tr[2];
      stereo_residual(d, y, obs, er);
      const double e2 = er[0] * er[0] * om[0] + er[1] * er[1] * om[1] + er[2] * er[2] * om[2];
      double r0 = e2, r1 = 1.;
      if (robust) huber(e2, delta, r0, r1);
      const double one[3] = {1., 1., 1.};
      double Jp[18], Ja[18], Js[9];
      edge_jacobians(d, R, tr, y, xa, ipz, 1., 1., one, Jp, Ja, Js);
      const bool self = ip == ia;   // J_pose + J_anchor = 0
      double vp[6];
#pragma unroll
      for (int r = 0; r < 6; ++r) vp[r] = self ? 0. : x[6 * ip + r];
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        double jv = Js[3 * q] * vl[0] + Js[3 * q + 1] * vl[1] + Js[3 * q + 2] * vl[2];
        if (!self) {
#pragma unroll
          for (int r = 0; r < 6; ++r) jv = fma(Jp[6 * q + r], vp[r], fma(Ja[6 * q + r], va[r], jv));
        }
        go[q] = -r1 * om[q] * jv;
        gw[q] = -r1 * er[q] * jv;
      }
      if (kCam) {   // de/df = -(y0, y1, y0 - b) / y2, de/dpx = -(1, 0, 1), de/dpy = -(0, 1, 0), de/db = (0, 0, f / y2)
        const double iz = 1. / y[2];
        gc[0] -= (y[0] * go[0] + y[1] * go[1] + (y[0] - d.b) * go[2]) * iz;
        gc[1] -= go[0] + go[2];
        gc[2] -= go[1];
        gc[3] += d.f * iz * go[2];
      }
    }
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      if (dobs) dobs[3 * (size_t)src + q] = go[q];
      if (dinfo) dinfo[3 * (size_t)src + q] = gw[q];
    }
  }
  if (kCam) {
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int s = LANES / 2; s > 0; s >>= 1) gc[q] += __shfl_xor_sync(gmask, gc[q], s);
    if (sub == 0)
#pragma unroll
      for (int q = 0; q < 4; ++q) cam_part[4 * (size_t)li + q] = gc[q];
  }
}

// One CTA: out[q] = sum over landmarks of part[l][q], each thread over a fixed stride of landmarks, then a fixed tree.
__global__ void __launch_bounds__(kGradThreads) k_grad_cam(const double* __restrict__ part, int L, double* __restrict__ out) {
  __shared__ double sh[4][kGradThreads];
  const int t = threadIdx.x;
  double s[4] = {0., 0., 0., 0.};
  for (int l = t; l < L; l += kGradThreads)
#pragma unroll
    for (int q = 0; q < 4; ++q) s[q] += __ldg(part + 4 * (size_t)l + q);
#pragma unroll
  for (int q = 0; q < 4; ++q) sh[q][t] = s[q];
  __syncthreads();
  for (int w = kGradThreads / 2; w > 0; w >>= 1) {
    if (t < w)
#pragma unroll
      for (int q = 0; q < 4; ++q) sh[q][t] += sh[q][t + w];
    __syncthreads();
  }
  if (t < 4) out[t] = sh[t][0];
}

// One thread per pose-pose constraint c (G2oEdgeSE3, e_c = log(T_ji T_i T_j^-1), cost e_c^T Lambda_c e_c), with the
// Jacobians of constraint_build: J_i = third(T_ji, e_c), J_j = -third(I, -e_c), zero for a fixed pose.  w = J_i v_i + J_j v_j;
//   dL/dLambda_c[a][b] = -(w_a e_b + w_b e_a) / 2   (symmetric: the cost sees Lambda_ab and Lambda_ba together)
//   dL/d delta_c       = -X^T Lambda_c w,  X = third(I, e_c) = de_c/d delta_c for T_ji <- exp(delta_c) T_ji
// X is the factor J_i already contains: third(T_ji, e) = third(I, e) Ad(T_ji), since T_ji exp(d) = exp(Ad(T_ji) d) T_ji
// puts a change of T_i in front of T_ji.  Both outputs of c are written by this thread alone.
__global__ void __launch_bounds__(kGradThreads)
k_grad_constraints(BaDev d, double* __restrict__ dcT, double* __restrict__ dcLam) {
  const int c = (int)(blockIdx.x * (unsigned)kGradThreads + threadIdx.x);
  if (c >= d.C) return;
  double w[6] = {0., 0., 0., 0., 0., 0.}, err[6] = {0., 0., 0., 0., 0., 0.};
  if (!d.ctl->chol_fail) {
    const double* pose = d.pose[d.ctl->cur];
    const int i = d.c_i[c], j = d.c_j[c];
    constraint_error(d, pose, c, err);
    const double I7[7] = {0, 0, 0, 1, 0, 0, 0};
    double J[36];
    if (!d.fixed[i]) {
      double T21[7];
      for (int k = 0; k < 7; ++k) T21[k] = d.c_T[7 * (size_t)c + k];
      third(T21, err, J);
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) w[a] += J[a * 6 + b] * d.x[6 * i + b];
    }
    if (!d.fixed[j]) {
      double md[6];
      for (int k = 0; k < 6; ++k) md[k] = -err[k];
      third(I7, md, J);
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) w[a] -= J[a * 6 + b] * d.x[6 * j + b];
    }
    if (dcT) {
      const double* Lm = d.c_Lam + 36 * (size_t)c;
      double u[6];
      for (int a = 0; a < 6; ++a) {
        double s = 0.;
        for (int b = 0; b < 6; ++b) s += Lm[a * 6 + b] * w[b];
        u[a] = s;
      }
      third(I7, err, J);
      for (int b = 0; b < 6; ++b) {
        double s = 0.;
        for (int a = 0; a < 6; ++a) s += J[a * 6 + b] * u[a];
        dcT[6 * (size_t)c + b] = -s;
      }
    }
  } else if (dcT) {
    for (int b = 0; b < 6; ++b) dcT[6 * (size_t)c + b] = 0.;
  }
  if (dcLam)
    for (int a = 0; a < 6; ++a)
      for (int b = 0; b < 6; ++b) dcLam[36 * (size_t)c + 6 * a + b] = -0.5 * (w[a] * err[b] + w[b] * err[a]);
}

template <int LANES>
void launch_edges(const BaDev& d, const int* list, int n, const double* g_psi, double lambda, int robust, double delta,
                  double* dobs, double* dinfo, double* cam_part, cudaStream_t st) {
  if (n <= 0) return;
  const long long threads = (long long)n * LANES;
  const unsigned grid = (unsigned)((threads + kGradThreads - 1) / kGradThreads);
  if (cam_part)
    k_grad_edges<LANES, true><<<grid, kGradThreads, 0, st>>>(d, list, n, g_psi, lambda, robust, delta, dobs, dinfo, cam_part);
  else
    k_grad_edges<LANES, false><<<grid, kGradThreads, 0, st>>>(d, list, n, g_psi, lambda, robust, delta, dobs, dinfo, nullptr);
}

}  // namespace

void launch_grad_rhs(const BaDev& d, const double* g_pose, const double* g_psi, double lambda, cudaStream_t st) {
  const long long threads = (long long)d.L + 6 * (long long)d.P;
  if (threads == 0) return;
  k_grad_rhs<<<(unsigned)((threads + kGradThreads - 1) / kGradThreads), kGradThreads, 0, st>>>(d, g_pose, g_psi, lambda);
}

// Tracks of up to kShortTrack slots: kShortLanes lanes each, over all landmarks; the longer ones (gen_lm: 9..32 slots
// or no observations, long_lm: more than 32) one warp each.
// cam_part [L][4] (nullptr: no camera term) holds each landmark's camera partial; dcam [4] their sum.
void launch_grad_edges(const BaDev& d, const double* g_psi, double lambda, int robust, double delta, double* dobs,
                       double* dinfo, double* cam_part, double* dcam, cudaStream_t st) {
  launch_edges<kShortLanes>(d, nullptr, d.L, g_psi, lambda, robust, delta, dobs, dinfo, cam_part, st);
  launch_edges<32>(d, d.gen_lm, d.ngen, g_psi, lambda, robust, delta, dobs, dinfo, cam_part, st);
  launch_edges<32>(d, d.long_lm, d.nlong, g_psi, lambda, robust, delta, dobs, dinfo, cam_part, st);
  if (cam_part) k_grad_cam<<<1, kGradThreads, 0, st>>>(cam_part, d.L, dcam);
}

void launch_grad_constraints(const BaDev& d, double* dcT, double* dcLam, cudaStream_t st) {
  if (d.C == 0 || (!dcT && !dcLam)) return;
  k_grad_constraints<<<(unsigned)((d.C + kGradThreads - 1) / kGradThreads), kGradThreads, 0, st>>>(d, dcT, dcLam);
}

}  // namespace svs
