// ba_dev.cuh -- device helpers shared by the BA kernels (edge residuals, small inverses,
// pose-pose constraint arithmetic).
#pragma once
#include "ba_types.cuh"
#include "se3_dev.cuh"

namespace svs {

// ------------------------------------------------------------------ helpers

__device__ __forceinline__ void load12(const double* __restrict__ Rt, int p, double R[9], double t[3]) {
  const double* q = Rt + 12 * (size_t)p;
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = __ldg(q + i);
  t[0] = __ldg(q + 9); t[1] = __ldg(q + 10); t[2] = __ldg(q + 11);
}

// T_ca = T_c * T_a^-1  as rotation + translation
__device__ __forceinline__ void rel_pose(const double Rc[9], const double tc[3], const double Ra[9],
                                         const double ta[3], double R[9], double t[3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      R[i * 3 + j] = Rc[i * 3] * Ra[j * 3] + Rc[i * 3 + 1] * Ra[j * 3 + 1] + Rc[i * 3 + 2] * Ra[j * 3 + 2];
#pragma unroll
  for (int i = 0; i < 3; ++i) t[i] = tc[i] - (R[i * 3] * ta[0] + R[i * 3 + 1] * ta[1] + R[i * 3 + 2] * ta[2]);
}

// e = z - pi_stereo(y)   (G2oCameraParameters::stereocam_uvu_map, anchored_points.cpp:43-50)
// 1/a and sqrt(a) from the hardware approximations + two Newton steps (full double precision up to
// rounding; the library versions cost 20+ instructions each on the edge path)
__device__ __forceinline__ double fast_inv(double a) {
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(a));
  double e = fma(-a, y, 1.0);
  y = fma(y, e, y);
  e = fma(-a, y, 1.0);
  return fma(y, e, y);
}
__device__ __forceinline__ double fast_sqrt(double a) {   // a >= 0
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(a));
  const double h = 0.5 * a;
  y = fma(y, fma(-h * y, y, 0.5), y);
  y = fma(y, fma(-h * y, y, 0.5), y);
  return a > 0. ? a * y : 0.;
}

__device__ __forceinline__ void stereo_residual(const BaDev& d, const double y[3], const double obs[3], double e[3]) {
  const double iz = fast_inv(y[2]);
  e[0] = obs[0] - ((y[0] * iz) * d.f + d.px);
  e[1] = obs[1] - ((y[1] * iz) * d.f + d.py);
  e[2] = obs[2] - (((y[0] - d.b) * iz) * d.f + d.px);
}

// robust cost of one observation at (pose, anchor, psi)
__device__ __forceinline__ double edge_cost(const BaDev& d, const double* __restrict__ Rt, int ip, const double Ra[9],
                                            const double ta[3], const double xa[3], const double obs[3],
                                            const double om[3], int robust, double delta) {
  if (om[0] == 0. && om[1] == 0. && om[2] == 0.) return 0.;   // zero information (padding edges): no cost, whatever the projection
  double Rc[9], tc[3], R[9], t[3], y[3], e[3];
  load12(Rt, ip, Rc, tc);
  rel_pose(Rc, tc, Ra, ta, R, t);
  mat3_vec(R, xa, y);
  y[0] += t[0]; y[1] += t[1]; y[2] += t[2];
  stereo_residual(d, y, obs, e);
  const double e2 = e[0] * e[0] * om[0] + e[1] * e[1] * om[1] + e[2] * e[2] * om[2];
  if (!robust) return e2;
  double r0, r1;
  huber(e2, delta, r0, r1);
  return r0;
}

__device__ __forceinline__ void inv3_sym_lambda(const double* __restrict__ D6, double lambda, double Di[9]) {
  // (Hll + lambda I)^-1 by cofactors (Eigen's 3x3 inverse, as used by g2o's D->inverse())
  const double a00 = D6[0] + lambda, a01 = D6[1], a02 = D6[2], a11 = D6[3] + lambda, a12 = D6[4], a22 = D6[5] + lambda;
  const double c00 = a11 * a22 - a12 * a12, c01 = a12 * a02 - a01 * a22, c02 = a01 * a12 - a11 * a02;
  const double det = a00 * c00 + a01 * c01 + a02 * c02;
  const double id = 1. / det;
  Di[0] = c00 * id; Di[1] = c01 * id; Di[2] = c02 * id;
  Di[3] = Di[1];    Di[4] = (a00 * a22 - a02 * a02) * id; Di[5] = (a01 * a02 - a00 * a12) * id;
  Di[6] = Di[2];    Di[7] = Di[5]; Di[8] = (a00 * a11 - a01 * a01) * id;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- overlap timeline (SVS_SOLVE_TIMING=3, scripts/probes/overlap_timeline.py): when each block column of S is complete
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// ---- programmatic dependent launch (svs_ba_optimize's trials, DESIGN.md 5).  Every kernel of a trial waits for the
// whole previous kernel of the stream (completed, its memory visible) before it reads anything that kernel may write,
// and then lets the next kernel's CTAs be scheduled, so that they are resident and waiting when this one ends instead
// of being launched after it.  Both are no-ops for a kernel that was launched without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// One work item that writes into block column `col` (and its right-hand side) is complete (the caller fences its writes
// first); the moment the column's last item lands is stamped.
__device__ __forceinline__ void signal_column(const BaDev& d, int col, long long* ready_ns) {
  const int was = atomicAdd(d.col_done + col, 1);
  if (ready_ns && was + 1 == __ldg(d.col_need + col)) ready_ns[col] = (long long)global_ns();
}

// ------------------------------------------------------------------ pose-pose constraint (one thread)

__device__ inline void third(const double A[7], const double dd[6], double out[36]) {
  // anchored_points.cpp:207-215: Adj_A + 1/2 ad_d Adj_A + 1/12 ad_d^2 Adj_A,
  // ad_d = SE3::d_lieBracketab_by_d_a(d)
  double Adj[36], dl[36], t1[36];
  se3_adj(A, Adj);
  double hu[9], ho[9];
  hat3(dd, hu);
  hat3(dd + 3, ho);
#pragma unroll
  for (int i = 0; i < 36; ++i) dl[i] = 0;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      dl[i * 6 + j] = -ho[i * 3 + j];
      dl[i * 6 + 3 + j] = -hu[i * 3 + j];
      dl[(i + 3) * 6 + 3 + j] = -ho[i * 3 + j];
    }
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) {
      double s = 0;
      for (int k = 0; k < 6; ++k) s += dl[i * 6 + k] * Adj[k * 6 + j];
      t1[i * 6 + j] = s;
    }
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) {
      double s = 0;
      for (int k = 0; k < 6; ++k) s += dl[i * 6 + k] * t1[k * 6 + j];
      out[i * 6 + j] = Adj[i * 6 + j] + 0.5 * t1[i * 6 + j] + (1. / 12.) * s;
    }
}

__device__ inline void constraint_error(const BaDev& d, const double* __restrict__ pose, int c, double err[6]) {
  double T21[7], T1[7], T2[7], T2i[7], A[7], B[7];
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    T21[i] = d.c_T[7 * (size_t)c + i];
    T1[i] = pose[7 * (size_t)d.c_i[c] + i];
    T2[i] = pose[7 * (size_t)d.c_j[c] + i];
  }
  se3_inv(T2, T2i);
  se3_mul(T21, T1, A);
  se3_mul(A, T2i, B);
  se3_log(B, err);
}

__device__ inline double constraint_chi2(const BaDev& d, const double* __restrict__ pose, int c) {
  double err[6];
  constraint_error(d, pose, c, err);
  const double* Lm = d.c_Lam + 36 * (size_t)c;
  double chi = 0;
  for (int a = 0; a < 6; ++a)
    for (int b = 0; b < 6; ++b) chi += err[a] * Lm[a * 6 + b] * err[b];
  return chi;
}

// g2o BaseBinaryEdge::constructQuadraticForm for one G2oEdgeSE3
__device__ inline void constraint_build(const BaDev& d, const double* __restrict__ pose, int c) {
  const int i = d.c_i[c], j = d.c_j[c];
  double err[6], Ji[36], Jj[36], T21[7];
  constraint_error(d, pose, c, err);
#pragma unroll
  for (int k = 0; k < 7; ++k) T21[k] = d.c_T[7 * (size_t)c + k];
  third(T21, err, Ji);
  {
    const double I7[7] = {0, 0, 0, 1, 0, 0, 0};
    double md[6];
    for (int k = 0; k < 6; ++k) md[k] = -err[k];
    third(I7, md, Jj);
    for (int k = 0; k < 36; ++k) Jj[k] = -Jj[k];
  }
  if (d.fixed[i]) for (int k = 0; k < 36; ++k) Ji[k] = 0;
  if (d.fixed[j]) for (int k = 0; k < 36; ++k) Jj[k] = 0;
  const double* Lm = d.c_Lam + 36 * (size_t)c;
  double chi = 0, Oe[6];
  for (int a = 0; a < 6; ++a) {
    double s = 0;
    for (int b = 0; b < 6; ++b) { s += Lm[a * 6 + b] * err[b]; chi += err[a] * Lm[a * 6 + b] * err[b]; }
    Oe[a] = -s;
  }
  d.chi_c[c] = chi;
  const int tii = d.tbl[(size_t)i * d.P + i], tjj = d.tbl[(size_t)j * d.P + j], tij = d.tbl[(size_t)i * d.P + j];
  double* Sii = d.S + 36 * (size_t)(tii >> 1);
  double* Sjj = d.S + 36 * (size_t)(tjj >> 1);
  double* Sij = d.S + 36 * (size_t)(tij >> 1);
  const int tr = tij & 1;
  for (int a = 0; a < 6; ++a) {
    double AtO[6], BtO[6];
    for (int b = 0; b < 6; ++b) {
      double sa = 0, sb = 0;
      for (int k = 0; k < 6; ++k) { sa += Ji[k * 6 + a] * Lm[k * 6 + b]; sb += Jj[k * 6 + a] * Lm[k * 6 + b]; }
      AtO[b] = sa; BtO[b] = sb;
    }
    double bi = 0, bj = 0;
    for (int k = 0; k < 6; ++k) { bi += Ji[k * 6 + a] * Oe[k]; bj += Jj[k * 6 + a] * Oe[k]; }
    atomicAdd(d.bp + 6 * i + a, bi);
    atomicAdd(d.bp + 6 * j + a, bj);
    for (int b = 0; b < 6; ++b) {
      double sii = 0, sjj = 0, sij = 0;
      for (int k = 0; k < 6; ++k) {
        sii += AtO[k] * Ji[k * 6 + b];
        sjj += BtO[k] * Jj[k * 6 + b];
        sij += AtO[k] * Jj[k * 6 + b];
      }
      atomicAdd(Sii + a * 6 + b, sii);
      atomicAdd(Sjj + a * 6 + b, sjj);
      atomicAdd(Sij + (tr ? b * 6 + a : a * 6 + b), sij);   // rows <-> pose i unless transposed
    }
  }
}


// The three Jacobian blocks of G2oEdgeProjectPSI2UVU (anchored_points.cpp:148-189) at the camera point y = R x_a + t
// of an observation: Jp[3][6] wrt the observing pose, Ja[3][6] wrt the anchor pose, Js[3][3] wrt psi, row q scaled by
// sw[q]; zp / za (0 or 1) multiply the pose / anchor blocks.
__device__ __forceinline__ void edge_jacobians(const BaDev& d, const double R[9], const double t[3], const double y[3],
                                               const double xa[3], double ipz, double zp, double za, const double sw[3],
                                               double* __restrict__ Jp, double* __restrict__ Ja, double* __restrict__ Js) {
  // d_stereoproj_d_y (transformations.h:62-71): rows (a 0 c0) (0 a c1) (a 0 c2)
  const double iz = fast_inv(y[2]);
  const double a = d.f * iz;
  const double c0 = -(d.f * y[0]) * iz * iz, c1 = -(d.f * y[1]) * iz * iz, c2 = -(d.f * (y[0] - d.b)) * iz * iz;
  // J_pose = -Jcam [I | -hat(y)]  (anchored_points.cpp:187, transformations.h:73-80)
  Jp[0] = zp * sw[0] * -a;  Jp[1] = 0;                 Jp[2] = zp * sw[0] * -c0;
  Jp[3] = zp * sw[0] * (-c0 * y[1]);  Jp[4] = zp * sw[0] * (-a * y[2] + c0 * y[0]);  Jp[5] = zp * sw[0] * (a * y[1]);
  Jp[6] = 0;                Jp[7] = zp * sw[1] * -a;   Jp[8] = zp * sw[1] * -c1;
  Jp[9] = zp * sw[1] * (a * y[2] - c1 * y[1]);  Jp[10] = zp * sw[1] * (c1 * y[0]);  Jp[11] = zp * sw[1] * (-a * y[0]);
  Jp[12] = zp * sw[2] * -a; Jp[13] = 0;                Jp[14] = zp * sw[2] * -c2;
  Jp[15] = zp * sw[2] * (-c2 * y[1]); Jp[16] = zp * sw[2] * (-a * y[2] + c2 * y[0]); Jp[17] = zp * sw[2] * (a * y[1]);
  // J_anchor = Jcam R [I | -hat(x_a)]  (anchored_points.cpp:188)
  double M[9];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    M[j] = a * R[j] + c0 * R[6 + j];
    M[3 + j] = a * R[3 + j] + c1 * R[6 + j];
    M[6 + j] = a * R[j] + c2 * R[6 + j];
  }
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const double s = za * sw[q];
    Ja[q * 6 + 0] = s * M[q * 3 + 0];
    Ja[q * 6 + 1] = s * M[q * 3 + 1];
    Ja[q * 6 + 2] = s * M[q * 3 + 2];
    Ja[q * 6 + 3] = s * -(M[q * 3 + 1] * xa[2] - M[q * 3 + 2] * xa[1]);
    Ja[q * 6 + 4] = s * -(-M[q * 3 + 0] * xa[2] + M[q * 3 + 2] * xa[0]);
    Ja[q * 6 + 5] = s * -(M[q * 3 + 0] * xa[1] - M[q * 3 + 1] * xa[0]);
  }
  // J_psi = -Jcam d_Tinvpsi_d_psi (anchored_points.cpp:186, transformations.h:82-95)
  double N[9];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    N[i * 3 + 0] = R[i * 3 + 0] * ipz;
    N[i * 3 + 1] = R[i * 3 + 1] * ipz;
    N[i * 3 + 2] = -(y[i] - t[i]) * ipz;
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    Js[j] = -sw[0] * (a * N[j] + c0 * N[6 + j]);
    Js[3 + j] = -sw[1] * (a * N[3 + j] + c1 * N[6 + j]);
    Js[6 + j] = -sw[2] * (a * N[j] + c2 * N[6 + j]);
  }
}

// One observation edge: residual, robust weight and the three Jacobian blocks (edge_jacobians), each row scaled by
// sqrt(rho' * Omega_qq); Ee[3] = scaled error.  Returns the robust cost rho(e^T Omega e).
__device__ __forceinline__ double linearize_edge(const BaDev& d, const double* __restrict__ Rt, int e, int ip,
                                               const double Ra[9], const double ta[3], const double xa[3], double ipz,
                                               int fa, int robust, double delta, double* __restrict__ Jp,
                                               double* __restrict__ Ja, double* __restrict__ Js, double* __restrict__ Ee) {
  const double obs[3] = {__ldg(d.e_obs + e), __ldg(d.e_obs + (size_t)d.E + e), __ldg(d.e_obs + 2 * (size_t)d.E + e)};
  const double om[3] = {__ldg(d.e_w + e), __ldg(d.e_w + (size_t)d.E + e), __ldg(d.e_w + 2 * (size_t)d.E + e)};
  if (om[0] == 0. && om[1] == 0. && om[2] == 0.) {
    // zero information: the edge contributes nothing, and its projection (a padding edge names a frame that never
    // saw the point) must not be evaluated -- 0 x inf would poison the sums
#pragma unroll
    for (int i = 0; i < 18; ++i) { Jp[i] = 0.; Ja[i] = 0.; }
#pragma unroll
    for (int i = 0; i < 9; ++i) Js[i] = 0.;
    Ee[0] = Ee[1] = Ee[2] = 0.;
    return 0.;
  }
  double Rc[9], tc[3], R[9], t[3], y[3], er[3];
  load12(Rt, ip, Rc, tc);
  rel_pose(Rc, tc, Ra, ta, R, t);
  mat3_vec(R, xa, y);
  y[0] += t[0]; y[1] += t[1]; y[2] += t[2];
  stereo_residual(d, y, obs, er);
  const double e2 = er[0] * er[0] * om[0] + er[1] * er[1] * om[1] + er[2] * er[2] * om[2];
  double r0 = e2, r1 = 1.;
  if (robust) huber(e2, delta, r0, r1);
  const double sw[3] = {fast_sqrt(r1 * om[0]), fast_sqrt(r1 * om[1]), fast_sqrt(r1 * om[2])};   // sqrt(rho' Omega)
  edge_jacobians(d, R, t, y, xa, ipz, d.fixed[ip] ? 0. : 1., fa ? 0. : 1., sw, Jp, Ja, Js);
  Ee[0] = sw[0] * er[0];
  Ee[1] = sw[1] * er[1];
  Ee[2] = sw[2] * er[2];
  return r0;
}

}  // namespace svs
