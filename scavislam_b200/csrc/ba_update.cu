// ba_update.cu -- k_update (landmark back-substitution, point update, trial chi2, LM decision),
// k_chi2, k_prep.
#include "ba_dev.cuh"
#include "ba_kernels.cuh"

#include <mutex>

namespace svs {

bool device_needs_smem_optin(int slot, size_t bytes) {
  static size_t granted[64][4] = {};
  static std::mutex mu;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || slot < 0 || slot >= 4) return true;
  std::lock_guard<std::mutex> lk(mu);
  if (bytes <= granted[dev][slot]) return false;
  granted[dev][slot] = bytes;
  return true;
}

// ------------------------------------------------------------------ k_update (+ LM decision)

// g2o::OptimizationAlgorithmLevenberg::solve, the part after the linear solve: rho test, lambda
// update, accept (swap state buffers) or reject (keep), trial-loop and Terminate conditions.
__device__ void lm_decide(LmCtl* ctl, double chi_cur, double chi_new, double scale_pts) {
  const int fail = ctl->chol_fail;
  double currentChi = chi_cur;
  const double tempChi = fail ? 1.7976931348623157e308 : chi_new;
  if (ctl->iter == 0 && ctl->qmax == 0) ctl->chi_init = currentChi;
  double lambda = ctl->lambda, ni = ctl->ni;
  double rho = currentChi - tempChi;
  double scale = fail ? 0. : ctl->scale_pose + scale_pts;   // computeScale(): sum x (lambda x + b)
  scale += 1e-3;
  rho /= scale;
  int cur = ctl->cur;
  if (rho > 0 && isfinite(tempChi)) {
    const double u = 2 * rho - 1;
    double alpha = 1. - u * u * u;
    alpha = fmin(alpha, 2. / 3.);
    const double sf = fmax(1. / 3., alpha);
    lambda *= sf;
    ni = 2;
    currentChi = tempChi;
    cur ^= 1;
  } else {
    lambda *= ni;
    ni *= 2;
  }
  int qmax = ctl->qmax + 1;
  ctl->trials_total += 1;
  const int again = (rho < 0 && qmax < ctl->max_trials) ? 1 : 0;
  ctl->lambda = lambda; ctl->ni = ni; ctl->cur = cur; ctl->rho = rho;
  ctl->chi_cur = currentChi; ctl->chi_new = tempChi;
  ctl->again = again;
  if (!again) {
    const int it = ctl->iter;
    if (it < kMaxIters) { ctl->chi_iter[it] = currentChi; ctl->lambda_iter[it] = lambda; ctl->trials_iter[it] = qmax; }
    ctl->stop = (qmax == ctl->max_trials || rho == 0) ? 1 : 0;
    ctl->iter = it + 1;
    qmax = 0;
  }
  ctl->qmax = qmax;
}

constexpr int kLmLanes = 8;   // lanes per landmark in k_update

// sum over the kLmLanes lanes of a landmark's group; groups of one warp may sit in different branches,
// so the shuffle names only the group's own lanes
__device__ __forceinline__ double group_sum(double v, unsigned gmask) {
#pragma unroll
  for (int o = kLmLanes / 2; o > 0; o >>= 1) v += __shfl_xor_sync(gmask, v, o);
  return v;
}

template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
k_update(BaDev d, int robust, double delta, int n_lm_blocks, int defer_decision) {
  __shared__ double sPart[WARPS][3];
  __shared__ int sLast;
  pdl_wait();
  pdl_launch_dependents();
  LmCtl* ctl = d.ctl;
  if (ctl->max_iters > 0 && (ctl->stop || ctl->iter >= ctl->max_iters)) return;   // speculatively enqueued trial: nothing left to do
  if (threadIdx.x == 0) atomicCAS(&ctl->t_update_start, 0ull, global_ns());
  const int cur = ctl->cur, trial = 1 - cur;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // every CTA helps clearing the reduced system for the next build
  {
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, gn = (size_t)gridDim.x * blockDim.x;
    for (size_t i = gid; i < (size_t)d.nblk * 36; i += gn) d.S[i] = 0.;
    for (size_t i = gid; i < (size_t)6 * d.P; i += gn) { d.bp[i] = 0.; d.bc[i] = 0.; }
    for (size_t i = gid; i < (size_t)d.P; i += gn) d.col_done[i] = 0;   // (counted on the overlap timeline runs)
  }
  double part_cur = 0, part_new = 0, part_scale = 0;   // this warp's share (valid on lane 0)
  if ((int)blockIdx.x >= n_lm_blocks) {
    const int c = ((int)blockIdx.x - n_lm_blocks) * (WARPS * 32) + (int)threadIdx.x;
    double a = 0, b = 0;
    if (c < d.C) {
      b = constraint_chi2(d, d.pose[trial], c);
      d.chi_c_new[c] = b;
      a = d.chi_c[c];
    }
    part_cur = warp_sum(a);
    part_new = warp_sum(b);
  } else {
    // four landmarks per warp, eight lanes each (a track is ~6 observations: one warp per landmark
    // ran 4/5 of its lanes idle); longer tracks just take more rounds of the strided loops
    const int sub = lane & (kLmLanes - 1);
    const unsigned gmask = ((1u << kLmLanes) - 1u) << (lane & ~(kLmLanes - 1));
    const int li = ((int)blockIdx.x * WARPS + warp) * (32 / kLmLanes) + lane / kLmLanes;
    double g_cur = 0, g_new = 0, g_scale = 0;   // this landmark's share (valid on sub-lane 0)
    if (li < d.L) {
      const double lambda = ctl->lambda;
      const int e0 = d.lm_eptr[li], k = d.lm_eptr[li + 1] - e0;
      const int s0 = d.lm_sptr[li], K = d.lm_sptr[li + 1] - s0;
      const double* psi = d.psi[cur] + 3 * (size_t)li;
      double* psin = d.psi[trial] + 3 * (size_t)li;
      if (k == 0 || ctl->chol_fail) {
        if (sub < 3) psin[sub] = psi[sub];
        g_cur = (k == 0) ? 0. : d.chi_l[li];
      } else {
        g_cur = d.chi_l[li];
        const int off = d.lm_self[li] ? 0 : 1;
        const int ia = d.lm_anchor[li];
        // c = b_l - sum_slots B_s^T x_s
        double c3[3] = {0, 0, 0};
        for (int s = sub; s < K; s += kLmLanes) {
          const int p = (s == 0) ? ia : d.e_pose[e0 + s - off];
          const double* xs = d.x + 6 * p;
#pragma unroll
          for (int r = 0; r < 6; ++r) {
            const double xr = xs[r];
#pragma unroll
            for (int q = 0; q < 3; ++q) c3[q] -= d.W[(size_t)(r * 3 + q) * d.nslots + s0 + s] * xr;
          }
        }
#pragma unroll
        for (int q = 0; q < 3; ++q) c3[q] = group_sum(c3[q], gmask);
        const double* Dbl = d.Dbl + 12 * (size_t)li;
        const double bl[3] = {Dbl[6], Dbl[7], Dbl[8]};
        double Di[9];
        inv3_sym_lambda(Dbl, lambda, Di);
        const double cc[3] = {bl[0] + c3[0], bl[1] + c3[1], bl[2] + c3[2]};
        double dpsi[3], pn[3];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          dpsi[q] = Di[q * 3] * cc[0] + Di[q * 3 + 1] * cc[1] + Di[q * 3 + 2] * cc[2];
          pn[q] = psi[q] + dpsi[q];
        }
        if (sub < 3) psin[sub] = pn[sub];
        g_scale = dpsi[0] * (lambda * dpsi[0] + bl[0]) + dpsi[1] * (lambda * dpsi[1] + bl[1]) +
                  dpsi[2] * (lambda * dpsi[2] + bl[2]);
        // robust chi2 of this landmark's observations at the trial state
        const double* __restrict__ Rt = d.Rt[trial];
        double Ra[9], ta[3];
        load12(Rt, ia, Ra, ta);
        const double ipz = 1. / pn[2];
        const double xa[3] = {pn[0] * ipz, pn[1] * ipz, ipz};
        double chi = 0;
        for (int i = sub; i < k; i += kLmLanes) {
          const int e = e0 + i;
          const double obs[3] = {__ldg(d.e_obs + e), __ldg(d.e_obs + (size_t)d.E + e), __ldg(d.e_obs + 2 * (size_t)d.E + e)};
          const double om[3] = {__ldg(d.e_w + e), __ldg(d.e_w + (size_t)d.E + e), __ldg(d.e_w + 2 * (size_t)d.E + e)};
          chi += edge_cost(d, Rt, d.e_pose[e], Ra, ta, xa, obs, om, robust, delta);
        }
        g_new = group_sum(chi, gmask);
      }
    }
    // the warp's share: its landmarks in a fixed order
    part_cur = warp_sum(sub == 0 ? g_cur : 0.);
    part_new = warp_sum(sub == 0 ? g_new : 0.);
    part_scale = warp_sum(sub == 0 ? g_scale : 0.);
  }
  // CTA partials in a fixed order -> part[blockIdx][3]; the last CTA to finish reduces them
  if (lane == 0) { sPart[warp][0] = part_cur; sPart[warp][1] = part_new; sPart[warp][2] = part_scale; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, b = 0, c = 0;
    for (int w = 0; w < WARPS; ++w) { a += sPart[w][0]; b += sPart[w][1]; c += sPart[w][2]; }
    double* pp = d.part + 3 * (size_t)blockIdx.x;
    pp[0] = a; pp[1] = b; pp[2] = c;
    __threadfence();
    const unsigned ticket = atomicAdd(d.ticket, 1u);
    sLast = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (!sLast) return;
  __threadfence();
  // deterministic final reduction (fixed partition, fixed order)
  double acc[3] = {0, 0, 0};
  for (int i = threadIdx.x; i < (int)gridDim.x; i += WARPS * 32) {
    const double* pp = d.part + 3 * (size_t)i;
    acc[0] += __ldcg(pp); acc[1] += __ldcg(pp + 1); acc[2] += __ldcg(pp + 2);
  }
  __shared__ double sFin[WARPS * 32][3];
  sFin[threadIdx.x][0] = acc[0]; sFin[threadIdx.x][1] = acc[1]; sFin[threadIdx.x][2] = acc[2];
  __syncthreads();
  for (int w = WARPS * 16; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) {
      sFin[threadIdx.x][0] += sFin[threadIdx.x + w][0];
      sFin[threadIdx.x][1] += sFin[threadIdx.x + w][1];
      sFin[threadIdx.x][2] += sFin[threadIdx.x + w][2];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    *d.ticket = 0;
    ctl->ns_update += (long long)(global_ns() - ctl->t_update_start);
    ctl->t_update_start = 0;
    if (defer_decision) {   // sharded window: the totals are summed over ranks before the decision
      d.totals[0] = sFin[0][0]; d.totals[1] = sFin[0][1]; d.totals[2] = sFin[0][2];
    } else {
      lm_decide(ctl, sFin[0][0], sFin[0][1], sFin[0][2]);
    }
  }
}

__global__ void k_decide_deferred(BaDev d) {
  if (threadIdx.x == 0 && blockIdx.x == 0) lm_decide(d.ctl, d.totals[0], d.totals[1], d.totals[2]);
}
void launch_decide_deferred(const BaDev& d, cudaStream_t st) { k_decide_deferred<<<1, 32, 0, st>>>(d); }

void launch_update(const BaDev& d, int robust, double delta, int defer_decision, cudaStream_t st, int pdl) {
  constexpr int WARPS = 8;
  constexpr int kPerBlock = WARPS * (32 / kLmLanes);
  const int n_lm_blocks = (d.L + kPerBlock - 1) / kPerBlock;
  const int n_c_blocks = (d.C + WARPS * 32 - 1) / (WARPS * 32);
  int nb = n_lm_blocks + n_c_blocks;
  if (nb == 0) nb = 1;   // still clears the reduced system and takes the LM decision
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(nb, 1, 1);
  cfg.blockDim = dim3(WARPS * 32, 1, 1);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaLaunchKernelEx(&cfg, k_update<WARPS>, d, robust, delta, n_lm_blocks, defer_decision);
}
int update_grid_blocks(int L, int C) {
  constexpr int WARPS = 8;
  constexpr int kPerBlock = WARPS * (32 / kLmLanes);
  const int nb = (L + kPerBlock - 1) / kPerBlock + (C + WARPS * 32 - 1) / (WARPS * 32);
  return nb > 0 ? nb : 1;
}

// ------------------------------------------------------------------ k_chi2 (state cur)

template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
k_chi2(BaDev d, int robust, double delta, int n_lm_blocks) {
  const int cur = d.ctl->cur;
  if ((int)blockIdx.x >= n_lm_blocks) {
    const int c = ((int)blockIdx.x - n_lm_blocks) * (WARPS * 32) + (int)threadIdx.x;
    if (c < d.C) d.chi_c[c] = constraint_chi2(d, d.pose[cur], c);
    return;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int li = (int)blockIdx.x * WARPS + warp;
  if (li >= d.L) return;
  const int e0 = d.lm_eptr[li], k = d.lm_eptr[li + 1] - e0;
  double chi = 0;
  if (k > 0) {
    const double* __restrict__ Rt = d.Rt[cur];
    const double* psi = d.psi[cur] + 3 * (size_t)li;
    double Ra[9], ta[3];
    load12(Rt, d.lm_anchor[li], Ra, ta);
    const double ipz = 1. / psi[2];
    const double xa[3] = {psi[0] * ipz, psi[1] * ipz, ipz};
    for (int i = lane; i < k; i += 32) {
      const int e = e0 + i;
      const double obs[3] = {__ldg(d.e_obs + e), __ldg(d.e_obs + (size_t)d.E + e), __ldg(d.e_obs + 2 * (size_t)d.E + e)};
      const double om[3] = {__ldg(d.e_w + e), __ldg(d.e_w + (size_t)d.E + e), __ldg(d.e_w + 2 * (size_t)d.E + e)};
      chi += edge_cost(d, Rt, d.e_pose[e], Ra, ta, xa, obs, om, robust, delta);
    }
    chi = warp_sum(chi);
  }
  if (lane == 0) d.chi_l[li] = chi;
}

void launch_chi2(const BaDev& d, int robust, double delta, cudaStream_t st) {
  constexpr int WARPS = 8;
  const int n_lm_blocks = (d.L + WARPS - 1) / WARPS;
  const int n_c_blocks = (d.C + WARPS * 32 - 1) / (WARPS * 32);
  if (n_lm_blocks + n_c_blocks == 0) return;
  k_chi2<WARPS><<<n_lm_blocks + n_c_blocks, WARPS * 32, 0, st>>>(d, robust, delta, n_lm_blocks);
}

// ------------------------------------------------------------------ k_prep: quaternion poses -> R,t

__global__ void k_prep(BaDev d, int buf) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= d.P) return;
  double T[7], R[9];
#pragma unroll
  for (int r = 0; r < 7; ++r) T[r] = d.pose[buf][7 * (size_t)p + r];
  quat_to_R(T, R);
#pragma unroll
  for (int r = 0; r < 9; ++r) d.Rt[buf][12 * (size_t)p + r] = R[r];
  d.Rt[buf][12 * (size_t)p + 9] = T[4];
  d.Rt[buf][12 * (size_t)p + 10] = T[5];
  d.Rt[buf][12 * (size_t)p + 11] = T[6];
}

// ------------------------------------------------------------------ k_regroup: user edge order -> internal SoA
// raw = [E][3] observations followed by [E][3] weights as the caller passed them; the internal order groups
// the edges of a landmark (set_problem), stored [3][E] so that a wave of edges reads coalesced
__global__ void k_regroup(BaDev d, const double* __restrict__ raw) {
  const int at = blockIdx.x * blockDim.x + threadIdx.x;
  if (at >= d.E) return;
  const int src = d.edge_src[at];
  if (src < 0) {   // padding edge of a completed track (set_problem): weight zero, observation irrelevant
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      d.e_obs_w[(size_t)q * d.E + at] = 0.;
      d.e_w_w[(size_t)q * d.E + at] = 0.;
    }
    return;
  }
  const size_t e = (size_t)src;
  const double* o = raw + 3 * e;
  const double* w = raw + 3 * (size_t)d.E_user + 3 * e;
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    d.e_obs_w[(size_t)q * d.E + at] = o[q];
    d.e_w_w[(size_t)q * d.E + at] = w[q];
  }
}
void launch_regroup(const BaDev& d, const double* raw, cudaStream_t st) {
  if (d.E > 0) k_regroup<<<(d.E + 255) / 256, 256, 0, st>>>(d, raw);
}

// ------------------------------------------------------------------ k_export: accepted state -> [P][7] poses, [L][3] psi in the CALLER's order
// (restoreDataFromG2o's read-out, slam_graph.cpp:1037-1058, as one contiguous buffer for a single device-to-host copy)
__global__ void k_export(BaDev d, double* __restrict__ out) {
  const int cur = d.ctl->cur;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 7 * d.P) out[i] = d.pose[cur][i];
  if (i < d.L) {
    const double* s = d.psi[cur] + 3 * (size_t)i;
    double* o = out + 7 * (size_t)d.P + 3 * (size_t)d.lm_user[i];
    o[0] = s[0]; o[1] = s[1]; o[2] = s[2];
  }
}
void launch_export(const BaDev& d, double* out, cudaStream_t st) {
  const int n = d.L > 7 * d.P ? d.L : 7 * d.P;
  if (n > 0) k_export<<<(n + 255) / 256, 256, 0, st>>>(d, out);
}

void launch_prep(const BaDev& d, int buf, cudaStream_t st) {
  if (d.P == 0) return;
  k_prep<<<(d.P + 127) / 128, 128, 0, st>>>(d, buf);
}
}  // namespace svs
