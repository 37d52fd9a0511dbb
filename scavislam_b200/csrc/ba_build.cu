// ba_build.cu -- k_build: fused linearise + J^T W J + 3x3 landmark elimination + Schur scatter.
//   G2oEdgeProjectPSI2UVU::computeError / linearizeOplus (anchored_points.cpp:148-189),
//   g2o BaseMultiEdge::constructQuadraticForm, BlockSolver<6,3>::buildSystem and the Schur part of
//   BlockSolver::solve -- one warp per landmark; the pose-pose constraints G2oEdgeSE3
//   (anchored_points.cpp:207-235) ride on trailing CTAs of the same launch.
#include "ba_dev.cuh"
#include "ba_kernels.cuh"

namespace svs {

// ------------------------------------------------------------------ k_build

// Per-warp shared-memory plan (doubles): per edge lane J~p[18] J~a[18] (stride 19), J~psi[9], e~[3];
// per slot B[18] Y[18] (stride 19); 16 scratch.  Then ints: pair table, slot poses.
constexpr int kSJ = 19;
__host__ __device__ inline int build_warp_doubles(int Kmax) { return (2 * kSJ + 12) * Kmax + 2 * kSJ * Kmax + 16; }
__host__ __device__ inline int build_warp_ints(int Kmax) { return ((Kmax * (Kmax + 1) / 2 + Kmax + 1) / 2) * 2; }
size_t build_smem_bytes(int warps, int Kmax) {
  return (size_t)warps * ((size_t)build_warp_doubles(Kmax) * 8 + (size_t)build_warp_ints(Kmax) * 4);
}

template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
k_build(BaDev d, const int* __restrict__ lm_list, int n_list, int Kmax, int robust, double delta, int n_lm_blocks) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const LmCtl* __restrict__ ctl = d.ctl;
  if (ctl->max_iters > 0 && (ctl->stop || ctl->iter >= ctl->max_iters)) return;   // speculatively enqueued trial: nothing left to do
  const int cur = ctl->cur;
  if ((int)blockIdx.x >= n_lm_blocks) {   // pose-pose constraints, one thread each
    const int c = ((int)blockIdx.x - n_lm_blocks) * (WARPS * 32) + (int)threadIdx.x;
    if (c < d.C) constraint_build(d, d.pose[cur], c);
    return;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int idx = (int)blockIdx.x * WARPS + warp;
  if (idx >= n_list) return;
  const int li = lm_list ? lm_list[idx] : idx;
  const double lambda = ctl->lambda;

  const int wd = build_warp_doubles(Kmax);
  double* sm = reinterpret_cast<double*>(smem_raw) + (size_t)warp * wd;
  double* sJp = sm;                       // [k][19]
  double* sJa = sJp + kSJ * Kmax;         // [k][19]
  double* sJs = sJa + kSJ * Kmax;         // [k][9]
  double* sE = sJs + 9 * Kmax;            // [k][3]
  double* sB = sE + 3 * Kmax;             // [K][19]
  double* sY = sB + kSJ * Kmax;           // [K][19]
  double* sD = sY + kSJ * Kmax;           // 16: D(6) bl(3) Dinv? -> D6, bl3
  int* si = reinterpret_cast<int*>(reinterpret_cast<double*>(smem_raw) + (size_t)WARPS * wd) +
            (size_t)warp * build_warp_ints(Kmax);
  int* sPose = si;                        // [K]
  int* sPair = si + Kmax;                 // [npairs]

  const int e0 = d.lm_eptr[li], k = d.lm_eptr[li + 1] - e0;
  const int s0 = d.lm_sptr[li], K = d.lm_sptr[li + 1] - s0;
  double* Dbl = d.Dbl + 12 * (size_t)li;
  if (k == 0) {
    if (lane < 12) Dbl[lane] = 0;
    if (lane == 0) d.chi_l[li] = 0;
    return;
  }
  const int has_self = d.lm_self[li];
  const int off = has_self ? 0 : 1;       // slot of edge lane i is i + off
  const int ia = d.lm_anchor[li];
  const double* __restrict__ Rt = d.Rt[cur];
  const double* __restrict__ psi = d.psi[cur] + 3 * (size_t)li;

  double Ra[9], ta[3];
  load12(Rt, ia, Ra, ta);
  const double p0 = __ldg(psi), p1 = __ldg(psi + 1), p2 = __ldg(psi + 2);
  const double ipz = 1. / p2;
  const double xa[3] = {p0 * ipz, p1 * ipz, ipz};   // invert_depth (maths_utils.h:66-69)
  const int fa = d.fixed[ia];

  double chi = 0;
  if (lane == 0) sPose[0] = ia;
  if (lane < k) {
    const int e = e0 + lane;
    const int ip = d.e_pose[e];
    sPose[lane + off] = ip;   // for the self edge (lane 0, off 0) this rewrites the anchor
    chi = linearize_edge(d, Rt, e, ip, Ra, ta, xa, ipz, fa, robust, delta, sJp + kSJ * lane, sJa + kSJ * lane,
                         sJs + 9 * lane, sE + 3 * lane);
    const double* Jp = sJp + kSJ * lane;
    const double* Js = sJs + 9 * lane;
    // own Hpl block B = J~p^T J~psi (6x3); the self edge's block is cancelled by its anchor part
    if (!(has_self && lane == 0)) {
      double* B = sB + kSJ * (lane + off);
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
          B[r * 3 + c] = Jp[r] * Js[c] + Jp[6 + r] * Js[3 + c] + Jp[12 + r] * Js[6 + c];
    }
  }
  chi = warp_sum(chi);
  if (lane == 0) d.chi_l[li] = chi;
  // pair table: (dst block, transpose, m, n) for all slot pairs m <= n
  __syncwarp();
  const int npairs = K * (K + 1) / 2;
  for (int pidx = lane; pidx < npairs; pidx += 32) {
    int m = 0, rem = pidx;
    while (rem >= K - m) { rem -= K - m; ++m; }
    const int n = m + rem;
    const int t = d.tbl[(size_t)sPose[m] * d.P + sPose[n]];
    sPair[pidx] = ((t >> 1) << 11) | ((t & 1) << 10) | (m << 5) | n;
  }
  // landmark sums: anchor Hpl block (18), Hll upper (6), b_l (3)
  const int i_first = has_self ? 1 : 0;   // first non-self edge lane
  if (lane < 27) {
    double s = 0;
    if (lane < 18) {
      const int r = lane / 3, c = lane % 3;
      for (int i = i_first; i < k; ++i)
        s += sJa[kSJ * i + r] * sJs[9 * i + c] + sJa[kSJ * i + 6 + r] * sJs[9 * i + 3 + c] +
             sJa[kSJ * i + 12 + r] * sJs[9 * i + 6 + c];
      sB[lane] = s;
    } else if (lane < 24) {
      const int t = lane - 18;
      const int r = t < 3 ? 0 : (t < 5 ? 1 : 2), c = t < 3 ? t : (t < 5 ? t - 2 : 2);
      for (int i = 0; i < k; ++i)
        s += sJs[9 * i + r] * sJs[9 * i + c] + sJs[9 * i + 3 + r] * sJs[9 * i + 3 + c] +
             sJs[9 * i + 6 + r] * sJs[9 * i + 6 + c];
      sD[t] = s;
    } else {
      const int c = lane - 24;
      for (int i = 0; i < k; ++i)
        s -= sJs[9 * i + c] * sE[3 * i] + sJs[9 * i + 3 + c] * sE[3 * i + 1] + sJs[9 * i + 6 + c] * sE[3 * i + 2];
      sD[6 + c] = s;
    }
  }
  __syncwarp();
  if (lane < 9) Dbl[lane] = sD[lane];
  double Di[9];
  inv3_sym_lambda(sD, lambda, Di);
  const double bl[3] = {sD[6], sD[7], sD[8]};
  // Y = B Dinv per slot; spill B to HBM (SoA) for the back-substitution
  for (int it = lane; it < K * 18; it += 32) {
    const int s = it / 18, rc = it % 18, r = rc / 3, c = rc % 3;
    const double* B = sB + kSJ * s + r * 3;
    sY[kSJ * s + rc] = B[0] * Di[c] + B[1] * Di[3 + c] + B[2] * Di[6 + c];
  }
  for (int c = 0; c < 18; ++c)
    if (lane < K) d.W[(size_t)c * d.nslots + s0 + lane] = sB[kSJ * lane + c];
  __syncwarp();
  // Schur scatter: for every slot pair, direct J^T W J part minus Y_m B_n^T
  const int skip_self = (d.flags & 1);
  const int total = npairs * 36;
  for (int fidx = lane; fidx < total; fidx += 32) {
    const int pidx = fidx / 36, el = fidx - pidx * 36;
    const int r = el / 6, c = el - r * 6;
    const int pk = sPair[pidx];
    const int m = (pk >> 5) & 31, n = pk & 31;
    const double* Ym = sY + kSJ * m + r * 3;
    const double* Bn = sB + kSJ * n + c * 3;
    double v = -(Ym[0] * Bn[0] + Ym[1] * Bn[1] + Ym[2] * Bn[2]);
    if (m == n) {
      if (m > 0) {
        const double* Jp = sJp + kSJ * (m - off);
        v += Jp[r] * Jp[c] + Jp[6 + r] * Jp[6 + c] + Jp[12 + r] * Jp[12 + c];
      } else {
        // anchor diagonal: all edges' J~a^T J~a; the self edge keeps g2o's J1^T W J1 (SURVEY 8c(4))
        for (int i = (skip_self ? i_first : 0); i < k; ++i) {
          const double* Ja = sJa + kSJ * i;
          v += Ja[r] * Ja[c] + Ja[6 + r] * Ja[6 + c] + Ja[12 + r] * Ja[12 + c];
        }
      }
    } else if (m == 0) {
      const double* Ja = sJa + kSJ * (n - off);
      const double* Jp = sJp + kSJ * (n - off);
      v += Ja[r] * Jp[c] + Ja[6 + r] * Jp[6 + c] + Ja[12 + r] * Jp[12 + c];
    }
    double* dst = d.S + 36 * (size_t)(pk >> 11) + (((pk >> 10) & 1) ? c * 6 + r : el);
    atomicAdd(dst, v);
  }
  // gradients: bp = -J^T W e, bc = Y b_l
  for (int it = lane; it < K * 6; it += 32) {
    const int s = it / 6, r = it - s * 6;
    double g = 0;
    if (s > 0) {
      const int i = s - off;
      g = -(sJp[kSJ * i + r] * sE[3 * i] + sJp[kSJ * i + 6 + r] * sE[3 * i + 1] + sJp[kSJ * i + 12 + r] * sE[3 * i + 2]);
    } else {
      for (int i = i_first; i < k; ++i)
        g -= sJa[kSJ * i + r] * sE[3 * i] + sJa[kSJ * i + 6 + r] * sE[3 * i + 1] + sJa[kSJ * i + 12 + r] * sE[3 * i + 2];
    }
    const double* Y = sY + kSJ * s + r * 3;
    const double corr = Y[0] * bl[0] + Y[1] * bl[1] + Y[2] * bl[2];
    const int p = sPose[s];
    atomicAdd(d.bp + 6 * p + r, g);
    atomicAdd(d.bc + 6 * p + r, corr);
  }
}

void launch_build_long(const BaDev& d, int robust, double delta, cudaStream_t st);

// Dispatch: landmark groups with <= 8 frames go to k_build_wave (ba_build_wave.cu); the rest (long
// tracks, landmarks without observations) and the pose-pose constraints to k_build.
void launch_build(const BaDev& d, int Kmax, int robust, double delta, cudaStream_t st) {
  constexpr int WARPS = 8;
  launch_build_wave(d, robust, delta, st);
  launch_build_long(d, robust, delta, st);
  const int n_lm_blocks = (d.ngen + WARPS - 1) / WARPS;
  const int n_c_blocks = 0;   // the pose-pose constraints ride on k_build_wave's launch
  const size_t smem = build_smem_bytes(WARPS, Kmax);
  if (device_needs_smem_optin(1, smem))
    cudaFuncSetAttribute(k_build<WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (n_lm_blocks + n_c_blocks == 0) return;
  k_build<WARPS><<<n_lm_blocks + n_c_blocks, WARPS * 32, smem, st>>>(d, d.gen_lm, d.ngen, Kmax, robust, delta, n_lm_blocks);
}

}  // namespace svs
