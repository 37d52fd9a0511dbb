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
// over the group by a butterfly, which leaves the same bits on every lane.
template <int LANES>
__global__ void __launch_bounds__(kGradThreads)
k_grad_edges(BaDev d, const int* __restrict__ list, int n, const double* __restrict__ g_psi, double lambda, int robust,
             double delta, double* __restrict__ dobs, double* __restrict__ dinfo) {
  const int lane = threadIdx.x & 31, sub = lane & (LANES - 1);
  const int idx = (int)((blockIdx.x * (unsigned)kGradThreads + threadIdx.x) / LANES);
  if (idx >= n) return;   // whole groups leave together
  const int li = list ? __ldg(list + idx) : idx;
  const int s0 = __ldg(d.lm_sptr + li), K = __ldg(d.lm_sptr + li + 1) - s0;
  if ((K > kShortTrack) != (LANES == 32)) return;   // the other instance's landmark
  const unsigned gmask = LANES == 32 ? 0xffffffffu : ((1u << LANES) - 1u) << (lane & ~(LANES - 1));
  const int e0 = __ldg(d.lm_eptr + li), k = __ldg(d.lm_eptr + li + 1) - e0;
  if (k == 0) return;
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
    }
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      if (dobs) dobs[3 * (size_t)src + q] = go[q];
      if (dinfo) dinfo[3 * (size_t)src + q] = gw[q];
    }
  }
}

template <int LANES>
void launch_edges(const BaDev& d, const int* list, int n, const double* g_psi, double lambda, int robust, double delta,
                  double* dobs, double* dinfo, cudaStream_t st) {
  if (n <= 0) return;
  const long long threads = (long long)n * LANES;
  k_grad_edges<LANES><<<(unsigned)((threads + kGradThreads - 1) / kGradThreads), kGradThreads, 0, st>>>(
      d, list, n, g_psi, lambda, robust, delta, dobs, dinfo);
}

}  // namespace

void launch_grad_rhs(const BaDev& d, const double* g_pose, const double* g_psi, double lambda, cudaStream_t st) {
  const long long threads = (long long)d.L + 6 * (long long)d.P;
  if (threads == 0) return;
  k_grad_rhs<<<(unsigned)((threads + kGradThreads - 1) / kGradThreads), kGradThreads, 0, st>>>(d, g_pose, g_psi, lambda);
}

// Tracks of up to kShortTrack slots: kShortLanes lanes each, over all landmarks; the longer ones (gen_lm: 9..32 slots
// or no observations, long_lm: more than 32) one warp each.
void launch_grad_edges(const BaDev& d, const double* g_psi, double lambda, int robust, double delta, double* dobs,
                       double* dinfo, cudaStream_t st) {
  launch_edges<kShortLanes>(d, nullptr, d.L, g_psi, lambda, robust, delta, dobs, dinfo, st);
  launch_edges<32>(d, d.gen_lm, d.ngen, g_psi, lambda, robust, delta, dobs, dinfo, st);
  launch_edges<32>(d, d.long_lm, d.nlong, g_psi, lambda, robust, delta, dobs, dinfo, st);
}

}  // namespace svs
