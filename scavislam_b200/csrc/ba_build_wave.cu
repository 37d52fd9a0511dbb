// ba_build_wave.cu -- k_build_wave: the fused linearise + J^T W J + landmark elimination + Schur
// scatter for landmark groups that share one (anchor, observer set) with at most 8 frames --
// the bulk of a SLAM window.  Same mathematics as k_build (ba_build.cu), different mapping:
//
//   * a warp owns a TASK: up to `chunk` consecutive landmarks with identical slot lists, so all
//     of them scatter into the same K(K+1)/2 blocks of the reduced camera system;
//   * edges are linearised 32 at a time (one lane per edge, several landmarks per wave), which
//     keeps every lane busy where one-warp-per-landmark leaves 3/4 of them idle;
//   * the task's whole contribution to the reduced system, S_task = sum_e G_e^T G_e - sum_l Y_l B_l^T (G_e the
//     3 x 6K scaled Jacobian of edge e over the task's slots, Y_l = B_l (Hll + lambda I)^-1, B_l the 6K x 3 Hpl stack),
//     is one FP64 tensor-core product (mma.m8n8k4.f64, DMMA) on 8 x 8 tiles of the 6K x 6K block, accumulated over
//     all landmarks of the task in the tile fragments and flushed with ONE set of RED.F64 per task instead of one
//     per landmark (the FP64 reduction rate, scripts/ubench/lat.cu, would make a per-landmark scatter a large share
//     of a launch).
//
// Reference semantics: G2oEdgeProjectPSI2UVU::linearizeOplus (anchored_points.cpp:168-189), g2o
// BaseMultiEdge::constructQuadraticForm, BlockSolver<6,3>::buildSystem / solve (Schur part).
#include <algorithm>
#include <cstdlib>

#include "ba_dev.cuh"
#include "ba_kernels.cuh"

namespace svs {

constexpr int kWvWarps = 4;
constexpr int kWvLm = 8;       // landmarks per wave
constexpr int kWvSlots = 40;   // slots per wave
constexpr int kWvJ = 19;       // row stride of the per-edge Jacobian rows (odd: conflict-free 64-bit stores)
constexpr int kWvLmD = 18;     // per-landmark scratch: D(6) bl(3) Dinv(9)
constexpr int kWvDoubles = 2 * 32 * kWvJ + 32 * 9 + 32 * 3 + 2 * kWvSlots * 18 + kWvLm * kWvLmD + 32;
constexpr int kWvInts = 8 + 40;   // slot poses, block table (36) padded
constexpr int kWvTiles = 6;       // 8-wide tiles over the 6K <= 48 rows / columns of a task's block
constexpr int kWvM = 56;          // row stride of the task's block staged for the flush
static_assert((8 * kWvTiles - 1) * kWvM + 8 * kWvTiles <= kWvDoubles && kWvDoubles % 2 == 0,
              "the staged block fits a warp's 16-byte aligned shared memory");

size_t build_wave_smem_bytes() { return (size_t)kWvWarps * (kWvDoubles * 8 + kWvInts * 4); }

// D += A B on one 8 x 8 tile, k = 4: lane holds A[lane >> 2][lane & 3], B[lane & 3][lane >> 2] and
// D[lane >> 2][2 (lane & 3) + {0, 1}]
__device__ __forceinline__ void dmma884(double& d0, double& d1, double a, double b) {
  asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
// upper tile pair (t1 <= t2) -> accumulator index
__host__ __device__ constexpr int tile_pair(int t1, int t2) { return t2 * (t2 + 1) / 2 + t1; }

// kTimeline: the overlap timeline's instance (SVS_SOLVE_TIMING=3, `timeline` = d.dbg + 160); the other one is the plain
// kernel, whose code the instrumentation must not touch
template <bool kTimeline>
__global__ void __launch_bounds__(kWvWarps * 32)
k_build_wave(BaDev d, int robust, double delta, int n_task_blocks, int prof, int persist, long long* timeline) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  if (!kTimeline) timeline = nullptr;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_wait();
  pdl_launch_dependents();
  const LmCtl* __restrict__ ctl = d.ctl;
  if (ctl->max_iters > 0 && (ctl->stop || ctl->iter >= ctl->max_iters)) return;   // speculatively enqueued trial: nothing left to do
  const int cur = ctl->cur;
  if (threadIdx.x == 0) atomicCAS(&d.ctl->t_build_start, 0ull, global_ns());
  // overlap timeline (SVS_SOLVE_TIMING=3): every finished task and constraint counts towards the readiness of its poses'
  // block columns (col_done); timeline[j] gets the moment column j became complete, timeline[2P] the first CTA's entry
  if (kTimeline && threadIdx.x == 0) atomicCAS(&d.ctl->t_build0, 0ull, global_ns());
  unsigned* const tctr = d.ticket + 1;
  // the last warp to leave resets the counter pair for the next launch (on the timeline runs every warp counts, and the
  // last one files the entry stamp)
  auto warp_exit = [&]() {
    if (!(persist || kTimeline)) return;
    if (kTimeline) __syncwarp();
    if (lane != 0) return;
    const unsigned nwarps_total = (unsigned)(kTimeline ? (int)gridDim.x : n_task_blocks) * kWvWarps;
    if (atomicAdd(tctr + 1, 1u) == nwarps_total - 1) {   // every other warp has drawn its last ticket
      tctr[0] = 0u; tctr[1] = 0u;
      if (kTimeline) timeline[2 * d.P] = (long long)atomicExch(&d.ctl->t_build0, 0ull);
    }
  };
  // pose-pose constraints (G2oEdgeSE3), one thread each, riding on CTAs of this launch so that their long
  // serial 6x6 arithmetic overlaps the landmark work instead of following it: the trailing CTAs of a
  // one-task-per-warp grid, the LEADING ones of a persistent grid (its task CTAs stay until the list is empty)
  {
    const int c_blocks = (int)gridDim.x - n_task_blocks;
    const int cb = persist ? (int)blockIdx.x : (int)blockIdx.x - n_task_blocks;
    if (cb >= 0 && cb < c_blocks) {
      const int c = cb * (kWvWarps * 32) + (int)threadIdx.x;
      if (c < d.C) {
        constraint_build(d, d.pose[cur], c);
        if (kTimeline) {
          __threadfence();
          signal_column(d, d.pos[d.c_i[c]], timeline);
          signal_column(d, d.pos[d.c_j[c]], timeline);
        }
      }
      if (kTimeline) warp_exit();
      return;
    }
  }
  // persistent grid: the warps draw tasks from one counter (longest tasks first, set_problem sorts them), so a
  // warp slot is never idle while tasks remain; the last warp to leave resets the counter pair for the next launch
  auto next_task = [&]() {
    int t = 0;
    if (lane == 0) t = (int)atomicAdd(tctr, 1u);
    return __shfl_sync(0xffffffffu, t, 0);
  };
  const double lambda = ctl->lambda;
  // (Drawing the next ticket early, when a task starts, hides the atomic's round trip, but a reserved task waits for
  //  its owner while other warps run dry at the end of the list; it was slower and is not done.)
  for (int task = persist ? next_task() : (int)blockIdx.x * kWvWarps + warp; task < d.ntasks;
       task = persist ? next_task() : d.ntasks) {
  double* sm = reinterpret_cast<double*>(smem_raw) + (size_t)warp * kWvDoubles;
  double* sJp = sm;
  double* sJa = sJp + 32 * kWvJ;
  double* sJs = sJa + 32 * kWvJ;
  double* sE = sJs + 32 * 9;
  double* sB = sE + 32 * 3;
  double* sY = sB + kWvSlots * 18;
  double* sLm = sY + kWvSlots * 18;
  double* sChi = sLm + kWvLm * kWvLmD;
  int* si = reinterpret_cast<int*>(reinterpret_cast<double*>(smem_raw) + (size_t)kWvWarps * kWvDoubles) + warp * kWvInts;
  int* sPose = si;
  int* sPair = si + 8;

  const int lm0 = d.task_lm[task], nlm = d.task_cnt[task];
  const int e_base = d.lm_eptr[lm0], k = d.lm_eptr[lm0 + 1] - e_base;
  const int s_base = d.lm_sptr[lm0], K = d.lm_sptr[lm0 + 1] - s_base;
  const int has_self = d.lm_self[lm0];
  const int off = has_self ? 0 : 1;
  const int i_first = has_self ? 1 : 0;
  const int ia = d.lm_anchor[lm0];
  const int fa = d.fixed[ia];
  const int skip_self = d.flags & 1;
  const double* __restrict__ Rt = d.Rt[cur];
  double Ra[9], ta[3];
  load12(Rt, ia, Ra, ta);

  // slot poses and the block table: sPair[tile_pair(m, n)] = (d.tbl entry (block << 1 | transpose) << 6) | m << 3 | n
  // for the slots m <= n
  if (lane == 0) sPose[0] = ia;
  if (lane < k && !(has_self && lane == 0)) sPose[lane + off] = d.e_pose[e_base + lane];
  __syncwarp();
  for (int p = lane; p < K * (K + 1) / 2; p += 32) {
    int n = 0;
    while (tile_pair(0, n + 1) <= p) ++n;
    const int m = p - tile_pair(0, n);
    sPair[p] = d.tbl[(size_t)sPose[m] * d.P + sPose[n]] << 6 | m << 3 | n;
  }
  __syncwarp();

  // the upper 8 x 8 tiles of the task's 6K x 6K block, as DMMA accumulator fragments
  const int ntiles = (6 * K + 7) / 8;
  double acc[tile_pair(0, kWvTiles)][2];
#pragma unroll
  for (int p = 0; p < tile_pair(0, kWvTiles); ++p) acc[p][0] = acc[p][1] = 0.;
  double accg[2] = {0., 0.}, accc[2] = {0., 0.};

  int nw_max = 32 / k;
  if (nw_max > kWvSlots / K) nw_max = kWvSlots / K;
  if (nw_max > kWvLm) nw_max = kWvLm;

  long long pacc[8] = {0, 0, 0, 0, 0, 0, 0, 0}, pclk = prof ? clock64() : 0;
#define PBW(i) do { if (prof) { __syncwarp(); const long long c_ = clock64(); pacc[i] += c_ - pclk; pclk = c_; } } while (0)
  PBW(0);
  for (int w0 = 0; w0 < nlm; w0 += nw_max) {
    const int nw = min(nw_max, nlm - w0);
    // ---- phase 1: one lane per edge of the wave
    double chi = 0.;
    if (lane < nw * k) {
      const int j = lane / k, i = lane - j * k;
      const int li = lm0 + w0 + j;
      const int e = e_base + (w0 + j) * k + i;
      const double* __restrict__ psi = d.psi[cur] + 3 * (size_t)li;
      const double p0 = __ldg(psi), p1 = __ldg(psi + 1), p2 = __ldg(psi + 2);
      const double ipz = fast_inv(p2);
      const double xa[3] = {p0 * ipz, p1 * ipz, ipz};
      const int ip = (has_self && i == 0) ? ia : sPose[i + off];
      double* Jp = sJp + kWvJ * lane;
      double* Js = sJs + 9 * lane;
      chi = linearize_edge(d, Rt, e, ip, Ra, ta, xa, ipz, fa, robust, delta, Jp, sJa + kWvJ * lane, Js, sE + 3 * lane);
      if (!(has_self && i == 0)) {   // own Hpl block B = J~p^T J~psi
        double* B = sB + 18 * (j * K + i + off);
#pragma unroll
        for (int r = 0; r < 6; ++r)
#pragma unroll
          for (int c = 0; c < 3; ++c) B[r * 3 + c] = Jp[r] * Js[c] + Jp[6 + r] * Js[3 + c] + Jp[12 + r] * Js[6 + c];
      }
    }
    sChi[lane] = chi;
    __syncwarp();
    PBW(1);
    if (lane < nw) {
      double s = 0.;
      for (int i = 0; i < k; ++i) s += sChi[lane * k + i];
      d.chi_l[lm0 + w0 + lane] = s;
    }
    // ---- phase 2: per-landmark sums over its edges: anchor Hpl block (18), Hll (6), b_l (3);
    //      one loop per kind so that the lanes of a round share a code path
    for (int it = lane; it < nw * 18; it += 32) {
      const int j = it / 18, t = it - j * 18, r = t / 3, c = t - r * 3;
      const double* Ja = sJa + kWvJ * (j * k + i_first);
      const double* Js = sJs + 9 * (j * k + i_first);
      double s = 0.;
      for (int i = i_first; i < k; ++i, Ja += kWvJ, Js += 9) s += Ja[r] * Js[c] + Ja[6 + r] * Js[3 + c] + Ja[12 + r] * Js[6 + c];
      sB[18 * (j * K) + t] = s;
    }
    for (int it = lane; it < nw * 6; it += 32) {
      const int j = it / 6, u = it - j * 6;
      const int r = u < 3 ? 0 : (u < 5 ? 1 : 2), c = u < 3 ? u : (u < 5 ? u - 2 : 2);
      const double* Js = sJs + 9 * (j * k);
      double s = 0.;
      for (int i = 0; i < k; ++i, Js += 9) s += Js[r] * Js[c] + Js[3 + r] * Js[3 + c] + Js[6 + r] * Js[6 + c];
      sLm[j * kWvLmD + u] = s;
    }
    for (int it = lane; it < nw * 3; it += 32) {
      const int j = it / 3, c = it - j * 3;
      const double* Js = sJs + 9 * (j * k);
      const double* Ee = sE + 3 * (j * k);
      double s = 0.;
      for (int i = 0; i < k; ++i, Js += 9, Ee += 3) s -= Js[c] * Ee[0] + Js[3 + c] * Ee[1] + Js[6 + c] * Ee[2];
      sLm[j * kWvLmD + 6 + c] = s;
    }
    __syncwarp();
    PBW(2);
    // ---- phase 3: (Hll + lambda I)^-1 per landmark; Hll / b_l to HBM for the back-substitution
    if (lane < nw) {
      double Di[9];
      inv3_sym_lambda(sLm + lane * kWvLmD, lambda, Di);
#pragma unroll
      for (int q = 0; q < 9; ++q) sLm[lane * kWvLmD + 9 + q] = Di[q];
    }
    for (int it = lane; it < nw * 9; it += 32) {
      const int j = it / 9, t = it - j * 9;
      d.Dbl[12 * (size_t)(lm0 + w0 + j) + t] = sLm[j * kWvLmD + t];
    }
    __syncwarp();
    // ---- phase 4: Y = B Dinv per slot; spill B (Hpl) to HBM, SoA over slots
    const int nslots_w = nw * K;
    for (int it = lane; it < nslots_w * 6; it += 32) {   // one row of a slot's block per lane
      const int sg = it / 6, r = it - sg * 6;
      const double* B = sB + 18 * sg + r * 3;
      const double* Di = sLm + (sg / K) * kWvLmD + 9;
      const double b0 = B[0], b1 = B[1], b2 = B[2];
      double* Y = sY + 18 * sg + r * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) Y[c] = b0 * Di[c] + b1 * Di[3 + c] + b2 * Di[6 + c];
    }
    {
      // (written as a double loop over (c, sg) with the address formed per element, this spill was the hottest source
      //  line of the kernel in a profiler capture.  A wave has at
      //  most 40 slots: two per lane, one pointer bumped by nslots per component, the 18 values of a slot read with
      //  16-byte shared-memory loads)
      const bool v0 = lane < nslots_w, v1 = lane + 32 < nslots_w;
      const double2* b0 = reinterpret_cast<const double2*>(sB + 18 * lane);
      const double2* b1 = reinterpret_cast<const double2*>(sB + 18 * (lane + 32));
      double* w = d.W + (size_t)s_base + (size_t)w0 * K + lane;
      const size_t ns = (size_t)d.nslots;
      if (v0) {
#pragma unroll
        for (int c = 0; c < 9; ++c) {
          const double2 t2 = b0[c];
          w[(size_t)(2 * c) * ns] = t2.x;
          w[(size_t)(2 * c + 1) * ns] = t2.y;
        }
      }
      if (v1) {
#pragma unroll
        for (int c = 0; c < 9; ++c) {
          const double2 t2 = b1[c];
          w[(size_t)(2 * c) * ns + 32] = t2.x;
          w[(size_t)(2 * c + 1) * ns + 32] = t2.y;
        }
      }
    }
    __syncwarp();
    PBW(3);
    // ---- phase 5: the wave's S_task terms on the tensor cores.  A lane's k-row is kb + (lane & 3), its column in tile t
    //      is 8 t + (lane >> 2): the A and B fragments of a tile load the same element of the k-row, so one value per
    //      lane and tile serves both operands.  k-rows past the wave's end, and columns past 6K, load zero.
    {
      const int kq = lane & 3, cl = lane >> 2;
      // G_e^T G_e, one slot at a time: the k-rows are (landmark, residual row) of the slot's edge; its row of G is
      // J~a in slot 0's columns (tile 0) and J~p in slot s's, so only the tiles of {0} and slot s take part.  The
      // self edge (slot 0) brings J~a alone -- g2o's J1^T W J1, SURVEY 8c(4) -- and nothing under the B5 skip.
#pragma unroll
      for (int s = 0; s < 8; ++s) {
        if (s >= K) break;
        if (s == 0 && (!has_self || skip_self)) continue;
        const int i = s == 0 ? 0 : s - off;
        for (int kb = 0; kb < 3 * nw; kb += 4) {
          const int kr = kb + kq, j = kr / 3, q = kr - 3 * j;
          const bool valid = kr < 3 * nw;
          const double* Ja = sJa + kWvJ * (j * k + i) + 6 * q;
          const double* Jp = sJp + kWvJ * (j * k + i) + 6 * q;
          double g[kWvTiles];
#pragma unroll
          for (int t = 0; t < kWvTiles; ++t) {
            const int col = 8 * t + cl;
            double v = 0.;
            if (t == 0 && col < 6) { if (valid) v = Ja[col]; }
            else if (s > 0 && col >= 6 * s && col < 6 * s + 6) { if (valid) v = Jp[col - 6 * s]; }
            g[t] = v;
          }
#pragma unroll
          for (int t2 = 0; t2 < kWvTiles; ++t2) {
            const bool in2 = t2 == 0 || t2 == 6 * s / 8 || t2 == (6 * s + 5) / 8;
#pragma unroll
            for (int t1 = 0; t1 <= t2; ++t1) {
              const bool in1 = t1 == 0 || t1 == 6 * s / 8 || t1 == (6 * s + 5) / 8;
              if (s > 0 && in1 && in2) dmma884(acc[tile_pair(t1, t2)][0], acc[tile_pair(t1, t2)][1], g[t1], g[t2]);
              if (s == 0 && t1 == 0 && t2 == 0) dmma884(acc[0][0], acc[0][1], g[0], g[0]);
            }
          }
        }
      }
      // - Y B^T: the k-rows are (landmark, column of Hpl); slot n's block of landmark j holds B[r][q] at
      // sB + 18 (j K + n) + 3 r + q, i.e. column 6 n + r at sB + 18 j K + 3 (6 n + r) + q
      for (int kb = 0; kb < 3 * nw; kb += 4) {
        const int kr = kb + kq, j = kr / 3, q = kr - 3 * j;
        const bool valid = kr < 3 * nw;
        const int o = 18 * j * K + q;
        double fy[kWvTiles], fb[kWvTiles];
#pragma unroll
        for (int t = 0; t < kWvTiles; ++t) {
          const int col = 8 * t + cl;
          const bool ok = valid && col < 6 * K;
          fy[t] = ok ? -sY[o + 3 * col] : 0.;
          fb[t] = ok ? sB[o + 3 * col] : 0.;
        }
#pragma unroll
        for (int t2 = 0; t2 < kWvTiles; ++t2)
          if (t2 < ntiles) {
#pragma unroll
            for (int t1 = 0; t1 <= t2; ++t1) dmma884(acc[tile_pair(t1, t2)][0], acc[tile_pair(t1, t2)][1], fy[t1], fb[t2]);
          }
      }
    }
    PBW(4);
    // ---- phase 6: gradients bp = -J^T W e, bc = Y b_l
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int it = lane + 32 * q;
      if (it < K * 6) {
        const int s = it / 6, r = it - s * 6;
        for (int j = 0; j < nw; ++j) {
          double g = 0.;
          if (s > 0) {
            const int l = j * k + s - off;
            g = -(sJp[kWvJ * l + r] * sE[3 * l] + sJp[kWvJ * l + 6 + r] * sE[3 * l + 1] + sJp[kWvJ * l + 12 + r] * sE[3 * l + 2]);
          } else {
            for (int i = i_first; i < k; ++i) {
              const int l = j * k + i;
              g -= sJa[kWvJ * l + r] * sE[3 * l] + sJa[kWvJ * l + 6 + r] * sE[3 * l + 1] + sJa[kWvJ * l + 12 + r] * sE[3 * l + 2];
            }
          }
          const double* Y = sY + 18 * (j * K + s) + r * 3;
          const double* bl = sLm + j * kWvLmD + 6;
          accg[q] += g;
          accc[q] += Y[0] * bl[0] + Y[1] * bl[1] + Y[2] * bl[2];
        }
      }
    }
    __syncwarp();
    PBW(5);
  }
  // ---- flush: one RED.F64 per element of the upper block triangle for the whole task.  The tiles go through the
  //      warp's shared memory (free once the last wave is done; row stride kWvM, 16-byte stores without bank conflicts),
  //      so that consecutive lanes add into consecutive elements of a block.  An element of a diagonal block below the
  //      diagonal whose tile lies below the tile diagonal is read from its mirror image.
  {
    double* sM = sm;
#pragma unroll
    for (int t2 = 0; t2 < kWvTiles; ++t2)
#pragma unroll
      for (int t1 = 0; t1 <= t2; ++t1)
        if (t2 < ntiles)
          *reinterpret_cast<double2*>(sM + (8 * t1 + (lane >> 2)) * kWvM + 8 * t2 + 2 * (lane & 3)) =
              make_double2(acc[tile_pair(t1, t2)][0], acc[tile_pair(t1, t2)][1]);
    __syncwarp();
    for (int e = lane; e < 36 * (K * (K + 1) / 2); e += 32) {
      const int p = e / 36, w = e - 36 * p;
      const int pk = sPair[p], m = (pk >> 3) & 7, n = pk & 7, t = pk >> 6;
      const int tr = t & 1, r = tr ? w % 6 : w / 6, c = tr ? w / 6 : w % 6;
      const int row = 6 * m + r, col = 6 * n + c;
      atomicAdd(d.S + 36 * (size_t)(t >> 1) + w, (row >> 3) > (col >> 3) ? sM[col * kWvM + row] : sM[row * kWvM + col]);
    }
  }
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int it = lane + 32 * q;
    if (it < K * 6) {
      const int s = it / 6, r = it - s * 6;
      const int p = sPose[s];
      atomicAdd(d.bp + 6 * p + r, accg[q]);
      atomicAdd(d.bc + 6 * p + r, accc[q]);
    }
  }
  if (kTimeline) {   // the task's blocks and right-hand sides are complete: count it for each of its slot poses' columns
    __threadfence();
    __syncwarp();
    if (lane < K) signal_column(d, d.pos[sPose[lane]], timeline);
  }
  PBW(6);
  if (prof && lane == 0)
    for (int i = 0; i < 7; ++i) atomicAdd(reinterpret_cast<unsigned long long*>(d.dbg) + 48 + i, (unsigned long long)pacc[i]);
#undef PBW
    __syncwarp();   // the next task reuses this warp's shared-memory tables
  }
  warp_exit();
}

// resident CTAs of k_build_wave on the current device (occupancy x SM count), cached per device
static int build_wave_resident_ctas() {
  static int cache[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return 1 << 30;
  if (cache[dev] == 0) {
    int per_sm = 0, sms = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_build_wave<false>, kWvWarps * 32, build_wave_smem_bytes());
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cache[dev] = per_sm > 0 && sms > 0 ? per_sm * sms : 1 << 30;
  }
  return cache[dev];
}

void launch_build_wave(const BaDev& d, int robust, double delta, cudaStream_t st, int pdl) {
  if (d.ntasks == 0 && d.C == 0) return;
  static const int prof = getenv("SVS_BUILD_TIMING") ? 1 : 0;
  // the opt-in above 48 KB of dynamic shared memory is per device: handles may live on several GPUs of one process
  if (device_needs_smem_optin(0, build_wave_smem_bytes())) {
    cudaFuncSetAttribute(k_build_wave<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)build_wave_smem_bytes());
    cudaFuncSetAttribute(k_build_wave<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)build_wave_smem_bytes());
  }
  int task_blocks = (d.ntasks + kWvWarps - 1) / kWvWarps;
  const int c_blocks = (d.C + kWvWarps * 32 - 1) / (kWvWarps * 32);
  // persistent grid when the tasks outnumber the warp slots: as many task CTAs as are resident at once (255 registers
  // and 101 KB of shared memory per CTA: two per SM), tasks drawn from a counter; otherwise one task per warp
  const int resident = build_wave_resident_ctas();
  const int persist = task_blocks > resident ? 1 : 0;
  if (persist) task_blocks = resident;
  static const int timing = getenv("SVS_SOLVE_TIMING") ? atoi(getenv("SVS_SOLVE_TIMING")) : 0;
  long long* timeline = timing >= 3 ? d.dbg + 160 : nullptr;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(task_blocks + c_blocks, 1, 1);
  cfg.blockDim = dim3(kWvWarps * 32, 1, 1);
  cfg.dynamicSmemBytes = build_wave_smem_bytes();
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  if (timeline) cudaLaunchKernelEx(&cfg, k_build_wave<true>, d, robust, delta, task_blocks, prof, persist, timeline);
  else cudaLaunchKernelEx(&cfg, k_build_wave<false>, d, robust, delta, task_blocks, prof, persist, (long long*)nullptr);
}

}  // namespace svs
