// ba_solve.cu -- k_solve: block-sparse right-looking Cholesky of the reduced camera system
// S dx = bs, forward/backward solve and pose update, on a thread-block cluster of two CTAs.
//   replaces g2o::LinearSolverCSparse<Matrix6d>::solve (instantiated at slam_graph.cpp:55-60) and
//   G2oVertexSE3::oplusImpl (anchored_points.cpp:53-58).
//
// The factor is a latency chain of P block columns.  What bounds it is not HBM and not the tensor
// cores (6x6 blocks, FP64) but the dependent-instruction latency of the pivot chain
//     chol(D_j) -> L_{j+1,j} = S_{j+1,j} L_jj^-T -> D_{j+1} -= L_{j+1,j} L_{j+1,j}^T -> chol(D_{j+1}) ...
// (per block column: 6 x [rsqrt + 2 Newton, multiply, fma] + the cross-block hand-over), so the kernel is organised around keeping that chain free of everything else:
//   * window-shaped pose graphs are factored from both ends at once ("twisted" / two-ended
//     elimination, ba_host.cu::choose_branches): each end is one CTA of a 2-CTA cluster with its own
//     SM (schedulers, shared-memory pipe, 227 KB), so the chain is P/2 + w columns long;
//   * in a CTA, warp 0 is the CHAIN warp and does nothing but the chain above, out of registers: every
//     lane factors the diagonal block redundantly (no shuffles between pivots), 21 lanes own one element
//     of the next diagonal block each and compute the two rows of L_{j+1,j} they need themselves;
//   * twelve HELPER warps (the ones that do not share the chain warp's scheduler) run one column behind:
//     scale the column's other rows, the trailing update in quarter-block units, the right-hand side
//     (forward solve rides along), and N_ij = L_ij L_jj^-1 for the backward pass.  Chain and helpers
//     meet only through two named barriers used as producer/consumer flags (bar.arrive / bar.sync):
//     "column j factored" and "column j's updates applied"; the chain waits on the second one column
//     late, so it is normally open;
//   * blocks live in a shared-memory ring over the next `cap` blocks in column-major order; updates of
//     the separator blocks go to a per-CTA accumulation area, and CTA 0 pulls CTA 1's area through
//     distributed shared memory before it factors the separator columns;
//   * backward: x_j = z_j - sum_i N_ij^T x_i with z = L^-T y and N folded in the forward pass, so a
//     column costs one shuffle broadcast and six FMAs on the chain; the separator solution is pushed
//     into CTA 1's shared memory.
// Graphs that are not banded enough for two ends run the same code as a single CTA (one chain).
#include <cooperative_groups.h>

#include <algorithm>
#include <cstdlib>
#include <mutex>

#include "ba_dev.cuh"
#include "ba_kernels.cuh"

namespace cg = cooperative_groups;

namespace svs {

constexpr int kSolveThreads = 384;               // 12 warps; warp w issues from scheduler w % 4
// Roles (factor_range).  Ten working warps (warps 8 and 11 idle through the factorisation): what bounds
// the helpers is the number of instructions their schedulers must issue per column (sixteen resident warps that all
// walked the column loop spent most of their issue slots on loop skeletons) and the FP64 pipe of a scheduler (two
// unit warps on one scheduler double the FMA phase).  Alternatives that were tried, fastest first:
//   this layout (unit warps 1-4, one per scheduler, warp 4 next to the chain)
//   fourth unit warp on warp 11 (scheduler 3, next to a unit warp and the urgent warp)
//   an earlier layout (unit warps 1, 2, 3, 5; row warps 6, 9; chain alone)
//   three unit warps, left-over units on the urgent warp
//   three unit warps, left-over units on the second row warp
constexpr int kChainWarp = 0;
constexpr int kUnitWarps = 4;                    // warps 1-4: quarter-block units of the trailing update
constexpr int kRowWarps = 2;                     // warps 5, 6: rows of the column, right-hand side
constexpr int kUrgentWarp = 7;                   // the two pair updates the chain reads next
constexpr int kNWarps = 2;                       // warps 9, 10: N rows for the backward pass (same schedulers as the row
                                                 // warps, so the instructions per scheduler hardly change)
__device__ __forceinline__ int unit_warp_index(int w) { return (w >= 1 && w <= 4) ? w - 1 : -1; }
__device__ __forceinline__ int row_warp_index(int w) { return w == 5 ? 0 : (w == 6 ? 1 : -1); }
__device__ __forceinline__ int n_warp_index(int w) { return w == 9 ? 0 : (w == 10 ? 1 : -1); }
constexpr int kUnitThreads = kUnitWarps * 32, kRowThreads = kRowWarps * 32, kNThreads = kNWarps * 32;
constexpr int kPubAll = 32 * (1 + kUnitWarps + kRowWarps + 1 + kNWarps);   // chain + unit + row + urgent + N warps
constexpr int kRowsAll = 32 * (kUnitWarps + kRowWarps + 1 + kNWarps);      // unit, row and N warps wait, row warps and urgent produce
constexpr int kRefillAll = 32 * (kUnitWarps + kRowWarps + kNWarps);       // the urgent warp only touches the next two columns: resident
constexpr int kUnitStride = kUnitThreads;
constexpr int kBarPub = 1;    // chain arrives, helpers + urgent warp sync: column j's diagonal factor is published
constexpr int kBarUrg = 2;    // urgent warp arrives, chain syncs: the chain's next inputs are up to date
constexpr int kBarH = 3;      // all rows of the column are scaled (row + urgent warps produce, unit + row warps wait)
constexpr int kBarH2 = 5;     // unit + row + N warps (ring refill)
constexpr int kBarBack = 4;   // backward pass, all threads of the CTA

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// 1/sqrt(a): hardware approximation (about 23 bits) + ONE third-order step, y1 = y0 (1 + e/2 + 3 e^2/8) with
// e = 1 - a y0^2 (error ~ 5/16 e^3 < 2^-64).  Dependent chain: approximation, 4 FP64 operations -- two Newton steps
// are 6, and the library rsqrt() carries special-case handling; this sits six times on the pivot chain of every column.
__device__ __forceinline__ double fast_rsqrt(double a) {
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(a));
  const double t = a * y;
  const double e = fma(-t, y, 1.0);
  const double ye = y * e;
  const double p = fma(0.375, e, 0.5);
  return fma(ye, p, y);
}

// Lower Cholesky of a 6x6 block given as its packed lower triangle a[r(r+1)/2 + c] (dlam added to the
// diagonal), in registers: l = packed lower factor, rinv = 1 / diagonal of the factor.
__device__ __forceinline__ bool chol6_packed(double a[21], double dlam, double l[21], double rinv[6]) {
#pragma unroll
  for (int r = 0; r < 6; ++r) a[r * (r + 1) / 2 + r] += dlam;
  bool ok = true;
#pragma unroll
  for (int c = 0; c < 6; ++c) {
    const double dv = a[c * (c + 1) / 2 + c];
    ok = ok && (dv > 0.);
    rinv[c] = fast_rsqrt(dv);
    l[c * (c + 1) / 2 + c] = dv * rinv[c];
#pragma unroll
    for (int r = c + 1; r < 6; ++r) l[r * (r + 1) / 2 + c] = a[r * (r + 1) / 2 + c] * rinv[c];
#pragma unroll
    for (int r = c + 1; r < 6; ++r)
#pragma unroll
      for (int c2 = c + 1; c2 <= r; ++c2)
        a[r * (r + 1) / 2 + c2] -= l[r * (r + 1) / 2 + c] * l[c2 * (c2 + 1) / 2 + c];
  }
  return ok;
}

// o = v L^-T (row vector): forward substitution against the packed lower factor
__device__ __forceinline__ void row_fwd(const double v[6], const double* __restrict__ L_, const double* __restrict__ ri,
                                        double o[6]) {
#pragma unroll
  for (int c = 0; c < 6; ++c) {
    double s = v[c];
#pragma unroll
    for (int q = 0; q < c; ++q) s = fma(-o[q], L_[c * (c + 1) / 2 + q], s);
    o[c] = s * ri[c];
  }
}
// n = o L^-1 (row vector): backward substitution
__device__ __forceinline__ void row_bwd(const double o[6], const double* __restrict__ L_, const double* __restrict__ ri,
                                        double n[6]) {
#pragma unroll
  for (int c = 5; c >= 0; --c) {
    double s = o[c];
#pragma unroll
    for (int q = c + 1; q < 6; ++q) s = fma(-n[q], L_[q * (q + 1) / 2 + c], s);
    n[c] = s * ri[c];
  }
}

__device__ __forceinline__ void load_row6(const double* __restrict__ p, double v[6]) {
  const double2* s2 = reinterpret_cast<const double2*>(p);
  const double2 s0 = s2[0], s1 = s2[1], s3 = s2[2];
  v[0] = s0.x; v[1] = s0.y; v[2] = s1.x; v[3] = s1.y; v[4] = s3.x; v[5] = s3.y;
}

// One contiguous range of columns factored by one CTA.
struct Team {
  int ring_off;               // (doubles into the dynamic shared memory) block id -> ring + ((id - org) & mask) * 36
  int org; unsigned mask;
  int cap;                    // ring capacity in blocks (refills keep [col_ptr[j], col_ptr[j] + cap) resident)
  int prefilled;              // 1: the whole range already lies in `ring` (separator phase)
  int j0, j1;                 // column range [j0, j1)
  int sep_blk0;               // updates of blocks >= sep_blk0 go to `area` (nblk when there is none)
  int area_off;               // separator accumulation area of this CTA: block b at area + (b - sep_blk0) * 36
  int slot;                   // index of the team's fail flags / diagonal-factor buffers
  int refill_period;
  long long* prof;            // nullptr or 16 cycle counters (developer knob SVS_SOLVE_TIMING=2)
  long long* timeline;        // nullptr or [P] %globaltimer when the chain publishes each column (SVS_SOLVE_TIMING=3)
};

#define TRACE(k, j) do { if (T.prof && T.slot == 0 && (j) - T.j0 >= 10 && (j) - T.j0 < 26 && (threadIdx.x & 31) == 0) T.prof[52 + (k) * 16 + ((j) - T.j0 - 10)] = clock64(); } while (0)
struct SolveShared {
  int yv_off;                 // right-hand side / solution, 6 doubles per column (offset into the dynamic shared memory)
  int* col_ptr; int* upd_ptr; int* row_idx;
  unsigned char* sfix;
  int (*fail)[2];
  double (*sL)[2][28];
  double* cdiag;
};

// Every shared-memory operand of the kernel is addressed relative to the one dynamic shared array, so that the
// compiler sees the address space (a select between pointers it cannot trace becomes a GENERIC load: an order of
// magnitude slower than LDS on this path).
extern __shared__ __align__(16) double sm_solve[];
__device__ __forceinline__ int ring_idx(const Team& T, int id) { return T.ring_off + (int)((unsigned)(id - T.org) & T.mask) * 36; }
#define ring_blk(T, id) (sm_solve + ring_idx(T, id))

// One quarter-block unit of the trailing update: rows 3h..3h+2, columns 3g..3g+2 of S_ab -= L_a L_b^T
// (18 16-byte loads, 54 FMAs).  u = 4 * pair + 2 h + g, ab = (a << 16) | b, dst = destination block.
// The address decode (indices only) is separate from the arithmetic so that the unit warps can do it while the
// column's rows are still being scaled.
struct UnitAddr {
  const double* la;      // 3 rows of L_a, 3 rows of L_b, the 3x3 destination (shared memory)
  const double* lb;
  double* dd;
  double* dg;            // destination in HBM when the block is not resident (else nullptr)
};
__device__ __forceinline__ UnitAddr unit_addr(const BaDev& d, const Team& T, int base, int hi, int u, int ab, int dst) {
  const int h = (u >> 1) & 1, g = u & 1;
  UnitAddr A;
  A.la = ring_blk(T, base + 1 + (ab >> 16)) + h * 18;
  A.lb = ring_blk(T, base + 1 + (ab & 0xffff)) + g * 18;
  const bool far = dst >= hi && dst < T.sep_blk0;   // not resident: read-modify-write in HBM
  A.dg = far ? d.S + (size_t)dst * 36 + h * 18 + g * 3 : nullptr;
  A.dd = sm_solve + (dst < hi ? ring_idx(T, dst) : T.area_off + (dst - T.sep_blk0) * 36) + h * 18 + g * 3;
  return A;
}
__device__ __forceinline__ void unit_run(const UnitAddr& A) {
  const double2* La = reinterpret_cast<const double2*>(A.la);
  const double2* Lb = reinterpret_cast<const double2*>(A.lb);
  double a[18], b[18], o[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) { const double2 v = La[q]; a[2 * q] = v.x; a[2 * q + 1] = v.y; }
#pragma unroll
  for (int q = 0; q < 9; ++q) { const double2 v = Lb[q]; b[2 * q] = v.x; b[2 * q + 1] = v.y; }
  double* Dg = A.dg;
  double* D = A.dd;
  if (Dg) {
#pragma unroll
    for (int rr = 0; rr < 3; ++rr)
#pragma unroll
      for (int cc = 0; cc < 3; ++cc) o[rr * 3 + cc] = Dg[rr * 6 + cc];
  } else {
#pragma unroll
    for (int rr = 0; rr < 3; ++rr)
#pragma unroll
      for (int cc = 0; cc < 3; ++cc) o[rr * 3 + cc] = D[rr * 6 + cc];
  }
#pragma unroll
  for (int rr = 0; rr < 3; ++rr)
#pragma unroll
    for (int cc = 0; cc < 3; ++cc)
#pragma unroll
      for (int k = 0; k < 6; ++k) o[rr * 3 + cc] = fma(-a[rr * 6 + k], b[cc * 6 + k], o[rr * 3 + cc]);
  if (Dg) {
#pragma unroll
    for (int rr = 0; rr < 3; ++rr)
#pragma unroll
      for (int cc = 0; cc < 3; ++cc) Dg[rr * 6 + cc] = o[rr * 3 + cc];
  } else {
#pragma unroll
    for (int rr = 0; rr < 3; ++rr)
#pragma unroll
      for (int cc = 0; cc < 3; ++cc) D[rr * 6 + cc] = o[rr * 3 + cc];
  }
}
__device__ __forceinline__ void quarter_unit(const BaDev& d, const Team& T, int base, int hi, int u, int ab, int dst) {
  unit_run(unit_addr(d, T, base, hi, u, ab, dst));
}

// Every refill_period columns the helpers (unit, row and urgent warps; `rid` in [0, kRefillAll)) reload the ring slots
// the finished columns freed.  Copies are never in flight while updates run, so a destination is either resident
// (< hi) or in HBM.
__device__ __forceinline__ void ring_refill(const BaDev& d, const Team& T, const int* col_ptr, int blk_end, int j, int rid,
                                            int& until_refill, int& hi) {
  if (--until_refill != 0) return;
  until_refill = T.refill_period;
  if (!(hi < blk_end && j + 1 < T.j1)) return;
  __threadfence();   // read-modify-writes of far blocks in HBM before the copies read them
  bar_sync(kBarH2, kRefillAll);
  const int hi_new = min(blk_end, col_ptr[j + 1] + T.cap);
  for (int cc = rid; cc < (hi_new - hi) * 18; cc += kRefillAll) {
    const int id = hi + cc / 18, w = cc % 18;
    cp_async16(ring_blk(T, id) + 2 * w, d.S + (size_t)id * 36 + 2 * w);
  }
  cp_async_commit();
  cp_async_wait_all();
  bar_sync(kBarH2, kRefillAll);
  hi = hi_new;
}

// Right-looking block Cholesky of columns [T.j0, T.j1); the forward solve rides along as an extra row.
//
// Three roles, three named barriers:
//   chain warp (warp 0)    factors D_c and publishes it (kBarPub, arrive); before it loads the inputs of column
//                          c+1 it waits for the URGENT updates of column c-1 (kBarUrg, sync);
//   urgent warp (warp 15)  after "column j published": scales the first two blocks of the column, (j+1, j) and
//                          (j+2, j) in a window, and applies the two pair updates the chain is going to read next
//                          -- D_{j+2} and S_{j+2,j+1} -- then signals (kBarUrg, arrive); less work than the
//                          chain's own column;
//   general helpers        everything else of column j: the other rows (L_ij) and the right-hand side (row warps), the
//                          other pair updates (unit warps), N_ij for the backward pass (N warps).  They re-join the chain only through kBarPub, one
//                          column later; since every helper must arrive there, "column j published" also means
//                          "all of column j-1 applied".
// kDiag: the chain warp also stores L_jj^-1 of every column it factors into d.Linv (row-major, zero above the
// diagonal: k_solve_general's layout), for the selected inversion of svs_chol6 (chol6_inv.cu)
template <bool kTimeline, bool kDiag>
__device__ void factor_range(const BaDev& d, const Team& T, const SolveShared& S, double lambda) {
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int* col_ptr = S.col_ptr; const int* upd_ptr = S.upd_ptr; const int* row_idx = S.row_idx;
  double* yv = sm_solve + S.yv_off;
  if (T.j0 >= T.j1) return;
  const int blk_end = col_ptr[T.j1];
  int hi = blk_end;
  if (!T.prefilled) {
    hi = min(blk_end, col_ptr[T.j0] + T.cap);
    for (int c = t; c < (hi - col_ptr[T.j0]) * 18; c += kSolveThreads) {
      const int id = col_ptr[T.j0] + c / 18, w = c % 18;
      cp_async16(ring_blk(T, id) + 2 * w, d.S + (size_t)id * 36 + 2 * w);
    }
    cp_async_commit();
    cp_async_wait_all();
  }
  __syncthreads();

  if (warp == kChainWarp) {
    // ------------------------------------------------------------------ the chain warp
    const int lr = (lane >= 1) + (lane >= 3) + (lane >= 6) + (lane >= 10) + (lane >= 15);
    const int r = lane < 21 ? lr : 0, c = lane < 21 ? lane - lr * (lr + 1) / 2 : 0;
    double dreg = ring_blk(T, col_ptr[T.j0])[r * 6 + c];
    double sr[6], sc[6], l[21], rinv[6];
    bool linked = false;
    int consumed = 0, produced = T.j1 - T.j0;
    long long pa[5] = {0, 0, 0, 0, 0}, pt = T.prof ? clock64() : 0;
#define PCH(i) do { if (T.prof) { const long long c_ = clock64(); pa[i] += c_ - pt; pt = c_; } } while (0)
    for (int j = T.j0; j < T.j1; ++j) {
      if (linked) {   // L_{j,j-1} rows r and c, then D_j[r][c] -= L_r . L_c
        double xr[6], xc[6];
        row_fwd(sr, l, rinv, xr);
        row_fwd(sc, l, rinv, xc);
        dreg -= (xr[0] * xc[0] + xr[1] * xc[1] + xr[2] * xc[2]) + (xr[3] * xc[3] + xr[4] * xc[4] + xr[5] * xc[5]);
      }
      if (lane < 21) S.cdiag[lane] = dreg;
      __syncwarp();
      PCH(0);
      // the inputs of the NEXT column, while this one is being factored: they are final once the urgent updates of
      // column j-1 are in (every older column is complete by then), and they must be read before column j is
      // published, because the helpers then overwrite S_{j+1,j} with L_{j+1,j}
      bool nlinked = false;
      const double* pD = nullptr;
      const double* pB = nullptr;
      if (j + 1 < T.j1) {
        const int base = col_ptr[j], nb = col_ptr[j + 1] - base - 1;
        nlinked = nb > 0 && row_idx[base + 1] == j + 1;
        pD = ring_blk(T, col_ptr[j + 1]) + r * 6 + c;
        pB = ring_blk(T, base + 1);
      }
      double2* sl2 = reinterpret_cast<double2*>(S.sL[T.slot][j & 1]);   // (addresses of the publish: formed before the
      int* pfail = &S.fail[T.slot][j & 1];                              //  factorisation, not behind the urgent barrier)
      double a[22];
      {
        const double2* c2 = reinterpret_cast<const double2*>(S.cdiag);
#pragma unroll
        for (int q = 0; q < 11; ++q) { const double2 v = c2[q]; a[2 * q] = v.x; a[2 * q + 1] = v.y; }
      }
      __syncwarp();
      // every lane factors the block redundantly in registers: no shuffles or shared-memory round trips
      // between the pivots (scripts/ubench/chol.cu)
      const bool ok = chol6_packed(a, lambda + (S.sfix[j] ? 1. : 0.), l, rinv);
      if (T.prof && l[20] != 0.) PCH(1);
      // the urgent updates of column j-1 (and with them everything older) are in: the next column's inputs are final
      if (j > T.j0) { bar_sync(kBarUrg, 64); ++consumed; }
      double dnext = 0.;
      if (pD) {
        dnext = *pD;
        if (nlinked) {
          load_row6(pB + r * 6, sr);
          load_row6(pB + c * 6, sc);
        }
      }
      if (T.prof && dnext != 1.2345e-300) { PCH(2); TRACE(1, j); }
      {   // publish l (21) and rinv (6): 14 independent 16-byte stores.  Every lane holds the same values and stores
          // them to the same addresses (one wavefront each): no divergent branch in front of the barrier arrival, and
          // no per-lane select of "its" element (a 27-deep dependent chain on the critical warp)
#pragma unroll
        for (int q = 0; q < 10; ++q) sl2[q] = make_double2(l[2 * q], l[2 * q + 1]);
        sl2[10] = make_double2(l[20], rinv[0]);
        sl2[11] = make_double2(rinv[1], rinv[2]);
        sl2[12] = make_double2(rinv[3], rinv[4]);
        sl2[13] = make_double2(rinv[5], 0.);
        if (!ok) *pfail = 1;
      }
      bar_arrive(kBarPub, kPubAll);
      TRACE(0, j);
      if (kTimeline && T.timeline && lane == 0) T.timeline[d.P + j] = (long long)global_ns();
      if (kDiag) {   // behind the publish: lane c < 6 forms column c of L_jj^-1 from l and rinv
        const int cc = lane < 6 ? lane : 0;
        double ai[6];
#pragma unroll
        for (int r2 = 0; r2 < 6; ++r2) {
          double v = r2 == cc ? 1. : 0.;
#pragma unroll
          for (int q = 0; q < r2; ++q) v = fma(-l[r2 * (r2 + 1) / 2 + q], ai[q], v);   // ai[q] = 0 above the diagonal
          ai[r2] = r2 < cc ? 0. : v * rinv[r2];
        }
        if (lane < 6)
#pragma unroll
          for (int r2 = 0; r2 < 6; ++r2) d.Linv[36 * (size_t)j + 6 * r2 + cc] = ai[r2];
      }
      PCH(3);
      if (!ok) { produced = j - T.j0; break; }
      linked = nlinked;
      dreg = dnext;
    }
    for (; consumed < produced; ++consumed) bar_sync(kBarUrg, 64);
    if (T.prof && lane == 0)
      for (int i = 0; i < 4; ++i) T.prof[i] = pa[i];
#undef PCH
  } else if (warp == kUrgentWarp) {
    // ------------------------------------------------------------------ the urgent warp
    // this lane's two output elements of the urgent updates: t < 21 -> packed lower element of D_{j+2}, else element
    // t - 21 of S_{j+2,j+1}
    auto decode = [](int t, int& r, int& c, bool& isS) {
      isS = t >= 21;
      if (isS) { r = (t - 21) / 6; c = (t - 21) - r * 6; }
      else { r = (t >= 1) + (t >= 3) + (t >= 6) + (t >= 10) + (t >= 15); c = t - r * (r + 1) / 2; }
    };
    int u0r, u0c, u1r, u1c;
    bool u0S, u1S;
    decode(lane, u0r, u0c, u0S);
    decode(min(lane + 32, 56), u1r, u1c, u1S);
    long long pu[4] = {0, 0, 0, 0}, ptu = T.prof ? clock64() : 0;
#define PUR(i) do { if (T.prof) { const long long c_ = clock64(); pu[i] += c_ - ptu; ptu = c_; } } while (0)
    for (int j = T.j0; j < T.j1; ++j) {
      const int base = col_ptr[j], nb = col_ptr[j + 1] - base - 1;
      const bool want = j + 2 < T.j1;   // the chain reads D_{j+2} and S_{j+2,j+1} next
      const int i1 = (j + 1 < T.j1 && nb > 0 && row_idx[base + 1] == j + 1) ? 0 : -1;   // index of row j+1 in the column (same
                                                                                        // rule as the chain's and the unit warps' `link`)
      int i2 = i1 + 1;                                                    // index of row j+2, if present
      if (!(i2 < nb && row_idx[base + 1 + i2] == j + 2)) i2 = -1;
      // every address below depends on the structure only: formed here, in the shadow of the wait for the diagonal
      // factor -- behind the barrier this warp is on the loop chain -> urgent -> chain, where only loads, FMAs and
      // stores remain
      const bool scale = lane < 6 * min(nb, 2);
      double* src = ring_blk(T, base + 1 + (scale ? lane / 6 : 0)) + (lane % 6) * 6;
      const double2* l2 = reinterpret_cast<const double2*>(S.sL[T.slot][j & 1]);
      const int* pfail = &S.fail[T.slot][j & 1];
      const bool urgent = want && i2 >= 0;
      const int nout = urgent ? (i1 >= 0 ? 57 : 21) : 0;
      const bool on0 = lane < nout, on1 = lane + 32 < nout;
      const double *pa0 = nullptr, *pb0 = nullptr, *pa1 = nullptr, *pb1 = nullptr;
      double *t0 = nullptr, *t1 = nullptr;
      if (urgent) {
        // D_{j+2} -= L2 L2^T (its 21 lower elements: the chain reads no others) and S_{j+2,j+1} -= L2 L1^T (36), ONE
        // element per lane and round: 6 loads, 6 dependent FMAs, one store
        const double* B2 = ring_blk(T, base + 1 + i2);
        const double* B1 = ring_blk(T, base + 1 + (i1 >= 0 ? i1 : i2));
        double* Dd = ring_blk(T, col_ptr[j + 2]);
        double* Sd = ring_blk(T, col_ptr[j + 1] + 1);
        pa0 = B2 + u0r * 6; pb0 = (u0S ? B1 : B2) + u0c * 6; t0 = (u0S ? Sd : Dd) + u0r * 6 + u0c;
        pa1 = B2 + u1r * 6; pb1 = (u1S ? B1 : B2) + u1c * 6; t1 = (u1S ? Sd : Dd) + u1r * 6 + u1c;
      }
      bar_sync(kBarPub, kPubAll);
      const int ufail = *pfail;
      if (T.prof && ufail >= 0) { PUR(0); TRACE(2, j); }
      if (ufail) break;
      // the first two blocks of the column are scaled here (the row warps take the others)
      if (scale) {
        double L_[28], v[6], o[6];
#pragma unroll
        for (int q = 0; q < 14; ++q) { const double2 t2 = l2[q]; L_[2 * q] = t2.x; L_[2 * q + 1] = t2.y; }
        load_row6(src, v);
        row_fwd(v, L_, L_ + 21, o);
        double2* d2 = reinterpret_cast<double2*>(src);
        d2[0] = make_double2(o[0], o[1]); d2[1] = make_double2(o[2], o[3]); d2[2] = make_double2(o[4], o[5]);
      }
      PUR(1);
      bar_arrive(kBarH, kRowsAll);   // (orders the stores above before the trailing update of the unit warps)
      if (urgent) {
        __syncwarp();   // the rows scaled above (other lanes) are visible
        double a0[6], b0[6], a1[6], b1[6];
        double o0 = 0., o1 = 0.;
        if (on0) { load_row6(pa0, a0); load_row6(pb0, b0); o0 = *t0; }
        if (on1) { load_row6(pa1, a1); load_row6(pb1, b1); o1 = *t1; }
        if (on0) {
#pragma unroll
          for (int k = 0; k < 6; ++k) o0 = fma(-a0[k], b0[k], o0);
          *t0 = o0;
        }
        if (on1) {
#pragma unroll
          for (int k = 0; k < 6; ++k) o1 = fma(-a1[k], b1[k], o1);
          *t1 = o1;
        }
      }
      PUR(2);
      TRACE(3, j);
      bar_arrive(kBarUrg, 64);
    }
    if (T.prof && lane == 0)
      for (int i = 0; i < 3; ++i) T.prof[12 + i] = pu[i];
#undef PUR
  } else if (unit_warp_index(warp) >= 0) {
    // ------------------------------------------------------------------ unit warps: the trailing update
    const int ut = unit_warp_index(warp) * 32 + lane;
    int until_refill = T.refill_period;
    long long ph[5] = {0, 0, 0, 0, 0}, pt = T.prof ? clock64() : 0;
#define PHL(i) do { if (T.prof) { const long long c_ = clock64(); ph[i] += c_ - pt; pt = c_; } } while (0)
    // Per column: indices (base, first update, number of units, the urgent warp's destinations) and this thread's
    // first (ab, dst) pair.  They depend on the structure only, so column j+1's are fetched while column j's rows are
    // being scaled (the unit warps have nothing else to do between the two barriers), and the first unit's addresses
    // are decoded there too: behind kBarH only loads, FMAs and stores remain.
    struct ColIdx { int base, u0, nunits, dU1, dU2; int2 e; };
    auto column_indices = [&](int j) {
      ColIdx c;
      const int nb = col_ptr[j + 1] - col_ptr[j] - 1;
      c.base = col_ptr[j];
      const int link = (j + 1 < T.j1 && nb > 0 && row_idx[c.base + 1] == j + 1) ? 1 : 0;
      c.u0 = upd_ptr[j] + link;
      c.nunits = (upd_ptr[j + 1] - c.u0) * 4;
      c.dU1 = c.dU2 = -1;   // destinations the urgent warp takes care of (same rule as there)
      if (j + 2 < T.j1 && link < nb && row_idx[c.base + 1 + link] == j + 2) {   // row j+2 can only sit right after row j+1
        c.dU1 = col_ptr[j + 2];
        if (link) c.dU2 = col_ptr[j + 1] + 1;
      }
      c.e = make_int2(0, 0);
      if (ut < c.nunits) c.e = make_int2(__ldg(d.upd_ab + c.u0 + (ut >> 2)), __ldg(d.upd_dst + c.u0 + (ut >> 2)));
      return c;
    };
    ColIdx cur = column_indices(T.j0 < T.j1 ? T.j0 : 0);
    for (int j = T.j0; j < T.j1; ++j) {
      bar_sync(kBarPub, kPubAll);   // (also: every helper is done with the previous column)
      const int col_failed = S.fail[T.slot][j & 1];   // (first read behind the barrier: the barrier wait ends here)
      if (T.prof && col_failed >= 0) { PHL(0); if (ut == 0) TRACE(4, j); }
      if (col_failed) break;
      const bool first = ut < cur.nunits && cur.e.y != cur.dU1 && cur.e.y != cur.dU2;
      UnitAddr A0 = {nullptr, nullptr, nullptr, nullptr};
      if (first) A0 = unit_addr(d, T, cur.base, hi, ut, cur.e.x, cur.e.y);
      ColIdx nxt = cur;
      if (j + 1 < T.j1) nxt = column_indices(j + 1);
      bar_sync(kBarH, kRowsAll);    // the column's rows are scaled
      if (T.prof && *reinterpret_cast<volatile int*>(&S.fail[T.slot][j & 1]) >= 0) PHL(1);
      // quarter-block units, at most one per thread for SLAM-shaped columns
      if (first) unit_run(A0);
      for (int u = ut + kUnitStride; u < cur.nunits; u += kUnitStride) {
        const int2 e = make_int2(__ldg(d.upd_ab + cur.u0 + (u >> 2)), __ldg(d.upd_dst + cur.u0 + (u >> 2)));
        if (e.y == cur.dU1 || e.y == cur.dU2) continue;   // the urgent warp's
        quarter_unit(d, T, cur.base, hi, u, e.x, e.y);
      }
      PHL(2);
      ring_refill(d, T, col_ptr, blk_end, j, ut, until_refill, hi);
      cur = nxt;
    }
    if (T.prof && ut == 8)
      for (int i = 0; i < 4; ++i) T.prof[4 + i] = ph[i];
#undef PHL
  } else if (row_warp_index(warp) >= 0) {
    // ------------------------------------------------------------------ row warps: L rows, right-hand side
    const int rt = row_warp_index(warp) * 32 + lane;
    int until_refill = T.refill_period;
    long long ph[5] = {0, 0, 0, 0, 0}, pt = T.prof ? clock64() : 0;
#define PHL(i) do { if (T.prof) { const long long c_ = clock64(); ph[i] += c_ - pt; pt = c_; } } while (0)
    for (int j = T.j0; j < T.j1; ++j) {
      const int base = col_ptr[j], nb = col_ptr[j + 1] - base - 1;
      const int nrows = nb * 6 + 1;
      // addresses first (structure only), in the shadow of the wait for the diagonal factor
      const int row0 = 6 * min(nb, 2) + rt;
      double* src0 = sm_solve + (row0 < nb * 6 ? ring_idx(T, base + 1 + row0 / 6) + (row0 % 6) * 6 : S.yv_off + 6 * j);
      const double* sl = S.sL[T.slot][j & 1];
      const int* pfail = &S.fail[T.slot][j & 1];
      bar_sync(kBarPub, kPubAll);
      const int col_failed = *pfail;
      if (T.prof && col_failed >= 0) PHL(0);
      if (col_failed) break;
      double L_[28];
      {
        const double2* l2 = reinterpret_cast<const double2*>(sl);
#pragma unroll
        for (int q = 0; q < 14; ++q) { const double2 t2 = l2[q]; L_[2 * q] = t2.x; L_[2 * q + 1] = t2.y; }
      }
      // ---- rows of the column: L_ij = S_ij L_jj^-T, kept in the ring for the trailing update (the first two blocks
      //      are the urgent warp's); the right-hand side is one more row (forward solve)
      for (int row = row0; row < nrows; row += kRowThreads) {
        double* src = row == row0 ? src0 : sm_solve + (row < nb * 6 ? ring_idx(T, base + 1 + row / 6) + (row % 6) * 6 : S.yv_off + 6 * j);
        double v[6], o[6];
        load_row6(src, v);
        row_fwd(v, L_, L_ + 21, o);
        double2* d2 = reinterpret_cast<double2*>(src);
        d2[0] = make_double2(o[0], o[1]); d2[1] = make_double2(o[2], o[3]); d2[2] = make_double2(o[4], o[5]);
      }
      PHL(1);
      bar_sync(kBarH, kRowsAll);
      if (T.prof && *reinterpret_cast<volatile int*>(&S.fail[T.slot][j & 1]) >= 0) PHL(2);
      // ---- b_a -= L_aj y_j
      for (int w = rt; w < nb * 6; w += kRowThreads) {
        const int a = w / 6, rr = w - a * 6;
        double La[6], yj[6];
        load_row6(ring_blk(T, base + 1 + a) + rr * 6, La);
        load_row6(yv + 6 * j, yj);
        const double sdot = (La[0] * yj[0] + La[1] * yj[1] + La[2] * yj[2]) + (La[3] * yj[3] + La[4] * yj[4] + La[5] * yj[5]);
        yv[6 * row_idx[base + 1 + a] + rr] -= sdot;
      }
      PHL(3);
      ring_refill(d, T, col_ptr, blk_end, j, kUnitThreads + rt, until_refill, hi);
    }
    if (T.prof && rt == 0)
      for (int i = 0; i < 4; ++i) T.prof[8 + i] = ph[i];
#undef PHL
  } else if (n_warp_index(warp) >= 0) {
    // ------------------------------------------------------------------ N warps: the folded factor for the backward pass
    // N_ij = L_ij L_jj^-1 (and z_j = y_j L_jj^-1), stored transposed in row-major order.  Nothing in the forward pass
    // waits for it, but every helper must be through a column before kBarPub opens for the next one: on warps of their
    // own these rows run beside the row warps' right-hand side instead of in front of it.
    const int nt = n_warp_index(warp) * 32 + lane;
    int until_refill = T.refill_period;
    for (int j = T.j0; j < T.j1; ++j) {
      const int base = col_ptr[j], nb = col_ptr[j + 1] - base - 1;
      const int nrows = nb * 6 + 1;
      const double* sl = S.sL[T.slot][j & 1];
      const int* pfail = &S.fail[T.slot][j & 1];
      bar_sync(kBarPub, kPubAll);
      // row-major position of the block of this thread's first row: a global load (an L2 round trip), in flight while
      // the rows are scaled.  Not issued before the barrier: its release would wait for it
      const int rpos0 = nt < nb * 6 ? __ldg(d.rowpos + base + 1 + nt / 6) : 0;
      if (*pfail) break;
      double L_[28];
      {
        const double2* l2 = reinterpret_cast<const double2*>(sl);
#pragma unroll
        for (int q = 0; q < 14; ++q) { const double2 t2 = l2[q]; L_[2 * q] = t2.x; L_[2 * q + 1] = t2.y; }
      }
      bar_sync(kBarH, kRowsAll);   // the column's rows are scaled
      for (int row = nt; row < nrows; row += kNThreads) {
        const double* src;
        double* gdst;
        int gstride;
        if (row < nb * 6) {
          const int a = row / 6, rr = row - a * 6;
          src = sm_solve + ring_idx(T, base + 1 + a) + rr * 6;
          const int rp = row == nt ? rpos0 : __ldg(d.rowpos + base + 1 + a);
          gdst = d.Nrow + (size_t)rp * 36 + rr;   // transposed inside the block
          gstride = 6;
        } else {
          src = sm_solve + S.yv_off + 6 * j;
          gdst = d.ywork + 6 * (size_t)j;
          gstride = 1;
        }
        double o[6], n[6];
        load_row6(src, o);
        row_bwd(o, L_, L_ + 21, n);
#pragma unroll
        for (int q = 0; q < 6; ++q) gdst[q * gstride] = n[q];
      }
      ring_refill(d, T, col_ptr, blk_end, j, kUnitThreads + kRowThreads + nt, until_refill, hi);
    }
  }
  __threadfence();   // N blocks and z (global) before the backward pass streams them back
  __syncthreads();
}

// Backward solve x_j = z_j - sum_{i > j} N_ij^T x_i, row oriented: the rows are walked from the last to the
// first; once x_i is final it is scattered into the columns of row i (c_j -= N_ij^T x_i for every block (i, j)).
// The row-major N blocks of a descending run of rows are ONE contiguous piece of memory; they are streamed through
// `buf` (2 x half blocks) in chunks of whole rows, double buffered: warp 0 walks the chain while the other warps
// fetch the next chunk.  Per row the chain is one shared-memory round trip (x_i) and six FMAs; no reduction across
// lanes, no shuffles.  Only blocks whose column lies in [c0, c1) are applied.
//
// A branch's pass walks two row ranges as one stream of chunks: the separator rows (x known, only scattered), then
// its own rows.  Positions v in [0, n) count up through [b0, b1) and then [a0, a1); the walk runs from n down to 0 and
// no chunk crosses from one range into the other.
constexpr int kMaxChunks = 48;
struct Walk {
  int a0, a1, b0, b1;   // rows [a0, a1) first, then [b0, b1)
  __device__ __forceinline__ int n() const { return (a1 - a0) + (b1 - b0); }
  __device__ __forceinline__ int row(int v) const { return v < b1 - b0 ? b0 + v : a0 + v - (b1 - b0); }
  __device__ __forceinline__ int floor(int v) const { return v > b1 - b0 ? b1 - b0 : 0; }   // lowest position of the
                                                                                           // range of position v - 1
};

// Chunk boundaries of the positions [0, top): top = b[0] > b[1] > ... (positions [b[k+1], b[k]) form chunk k: the
// longest run of whole rows of one range of at most `half` blocks, or one row if it is longer), at most kMaxChunks of
// them, their count in sChunk[kMaxChunks + 1].  One warp: the lanes test 32 candidate lower ends of a chunk at once
// (the block count of a run only grows as its lower end moves down, so the first lane that stops is the greedy end).
__device__ void plan_chunks(const int* rptr, const Walk& W, int top, int half, int* sChunk) {
  const int lane = threadIdx.x & 31;
  int n = 0, a = top;
  if (lane == 0) sChunk[0] = top;
  while (a > 0 && n < kMaxChunks) {
    const int lo = W.floor(a), end = rptr[W.row(a - 1) + 1];
    int b = lo;
    for (int base = a - 1;; base -= 32) {
      const int c = base - lane;
      const bool stop = c <= lo || end - rptr[W.row(c - 1)] > half;
      const unsigned m = __ballot_sync(0xffffffffu, stop);
      if (m) { b = base - (__ffs(m) - 1); break; }
    }
    ++n;
    if (lane == 0) sChunk[n] = b;
    a = b;
  }
  if (lane == 0) sChunk[kMaxChunks + 1] = n;
}

// Chunk k into its half of the buffer (cp.async, one commit group), by threads tid of nth.
__device__ __forceinline__ void load_chunk(const BaDev& d, const int* rptr, const Walk& W, const int* sChunk, int k,
                                           int buf_off, int half, int tid, int nth) {
  const int b0 = rptr[W.row(sChunk[k + 1])], n16 = (rptr[W.row(sChunk[k] - 1) + 1] - b0) * 18;
  double* dst = sm_solve + buf_off + (k & 1) * half * 36;
  const double* src = d.Nrow + (size_t)b0 * 36;
  for (int c = tid; c < n16; c += nth) cp_async16(dst + 2 * (size_t)c, src + 2 * (size_t)c);
  cp_async_commit();
}

// The first round of a backward pass (its chunk plan, and the first chunk in flight), so that a CTA can do it while it
// waits for the other one; scatter_rows(..., planned = true) then starts with the rows.
__device__ void plan_rows(const BaDev& d, const Walk& W, int top, int buf_off, int half, const SolveShared& S, int* sChunk) {
  if (threadIdx.x < 32) plan_chunks(S.upd_ptr, W, top, half, sChunk);
  bar_sync(kBarBack, kSolveThreads);
  if (top > 0) load_chunk(d, S.upd_ptr, W, sChunk, 0, buf_off, half, threadIdx.x, kSolveThreads);
}

// The pose update (G2oVertexSE3::oplusImpl) rides behind the backward pass: once a chunk of rows is done, x of its rows
// is final, and during the next chunk the warps that do not share warp 0's scheduler apply exp(dx) T of those rows
// into the trial buffer (pose and Rt of 1 - cur, and dx into d.x).  Row i is taken by pose thread i % kPoseThreads.
// A thread adds its rows' terms of scale = sum dx (lambda dx + b) into its own sum in the order it takes them (chunks in
// walking order, rows ascending inside a chunk); the threads' sums meet in the kernel's fixed reduction.  So the order
// is fixed by the structure alone.
constexpr int kPoseThreads = 9 * 32;
__device__ __forceinline__ int pose_thread(int warp, int lane) { return (warp & 3) ? (warp - (warp >> 2) - 1) * 32 + lane : -1; }
struct PoseTail {
  bool on_a, on_b;  // update the poses of the rows [a0, a1) / [b0, b1) of the walk
  double lambda;
  int cur;
};
struct PoseIn {     // what the update of row j reads besides x_j: fetched one chunk ahead
  int j, p;
  double b[6], T[7];
};
__device__ __forceinline__ void pose_load(const BaDev& d, int cur, int j, PoseIn& q) {
  q.j = j;
  q.p = d.perm[j];
#pragma unroll
  for (int rr = 0; rr < 6; ++rr) q.b[rr] = d.bp[6 * q.p + rr];
#pragma unroll
  for (int rr = 0; rr < 7; ++rr) q.T[rr] = d.pose[cur][7 * (size_t)q.p + rr];
}
__device__ __forceinline__ void pose_apply(const BaDev& d, const PoseIn& q, const double* xj, bool fixed, double lambda,
                                           int cur, double& sc) {
  const int p = q.p;
  double dx[6], Tn[7];
#pragma unroll
  for (int rr = 0; rr < 6; ++rr) {
    dx[rr] = fixed ? 0. : xj[rr];
    sc += dx[rr] * (lambda * dx[rr] + q.b[rr]);
  }
  if (fixed) {
#pragma unroll
    for (int rr = 0; rr < 7; ++rr) Tn[rr] = q.T[rr];
  } else {
    double dT[7];
    se3_exp(dx, dT);
    se3_mul(dT, q.T, Tn);
  }
  double R[9];
  quat_to_R(Tn, R);
#pragma unroll
  for (int rr = 0; rr < 6; ++rr) d.x[6 * p + rr] = dx[rr];
#pragma unroll
  for (int rr = 0; rr < 7; ++rr) d.pose[1 - cur][7 * (size_t)p + rr] = Tn[rr];
#pragma unroll
  for (int rr = 0; rr < 9; ++rr) d.Rt[1 - cur][12 * (size_t)p + rr] = R[rr];
  d.Rt[1 - cur][12 * (size_t)p + 9] = Tn[4];
  d.Rt[1 - cur][12 * (size_t)p + 10] = Tn[5];
  d.Rt[1 - cur][12 * (size_t)p + 11] = Tn[6];
}

__device__ void scatter_rows(const BaDev& d, const Walk& W, int c0, int c1, int buf_off, int half, const SolveShared& S,
                             int* sChunk, bool planned, const PoseTail& pt, double& sc) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int* rptr = S.upd_ptr;   // the forward pass's index arrays have been replaced by the row-major ones
  const int* rcol = S.row_idx;
  double* xv = sm_solve + S.yv_off;
  const int r = lane % 6, g = lane / 6;   // five lane groups take the blocks of a row; lanes 30, 31 idle
  const int pw = (pt.on_a || pt.on_b) ? pose_thread(warp, lane) : -1;
  PoseIn pin;
  pin.j = -1;
  // the rows [lo, hi) of chunk k, whether their poses are updated, this pose thread's first row there (or one past the
  // chunk), and the update of every one of its rows there
  auto chunk_rows = [&](int k, int& lo, int& hi) { lo = W.row(sChunk[k + 1]); hi = W.row(sChunk[k] - 1) + 1; };
  auto chunk_poses = [&](int k) { return sChunk[k + 1] >= W.b1 - W.b0 ? pt.on_a : pt.on_b; };
  auto first_row = [&](int lo) { return lo + (pw - lo % kPoseThreads + kPoseThreads) % kPoseThreads; };
  auto poses_of = [&](int k) {
    if (!chunk_poses(k)) return;
    int lo, hi;
    chunk_rows(k, lo, hi);
    for (int i = first_row(lo); i < hi; i += kPoseThreads) {
      if (i != pin.j) pose_load(d, pt.cur, i, pin);
      pose_apply(d, pin, xv + 6 * i, S.sfix[i], pt.lambda, pt.cur, sc);
    }
  };
  for (int top = W.n(); top > 0; planned = false) {
    if (!planned) plan_rows(d, W, top, buf_off, half, S, sChunk);
    cp_async_wait_all();
    bar_sync(kBarBack, kSolveThreads);
    const int nchunks = sChunk[kMaxChunks + 1];
    for (int k = 0; k < nchunks; ++k) {
      if (k + 1 < nchunks && warp > 0) load_chunk(d, rptr, W, sChunk, k + 1, buf_off, half, t - 32, kSolveThreads - 32);
      if (warp == 0) {
        const double* b = sm_solve + buf_off + (k & 1) * half * 36;
        int rlo, rhi;
        chunk_rows(k, rlo, rhi);
        const int b0 = rptr[rlo];
        // Software pipeline: everything of a row that does not depend on x -- its block range, this lane's first
        // block (column and the N row) -- is fetched while the previous row is being scattered; what is left on the
        // chain per row is the read of x_i, six FMAs and the read-modify-write of the target column.
        int i = rhi - 1;
        int p0 = 0, nb = 0, col = -1, colB = -1;
        double Nt[6] = {0, 0, 0, 0, 0, 0}, NtB[6] = {0, 0, 0, 0, 0, 0};
        auto prefetch = [&](int row) {   // two blocks per lane group (g and g + 5): a window row has 7-8 blocks
          p0 = rptr[row]; nb = rptr[row + 1] - p0; col = -1; colB = -1;
          if (lane < 30) {
            if (g < nb) {
              col = rcol[p0 + g];
              load_row6(b + (size_t)(p0 - b0 + g) * 36 + r * 6, Nt);
            }
            if (g + 5 < nb) {
              colB = rcol[p0 + g + 5];
              load_row6(b + (size_t)(p0 - b0 + g + 5) * 36 + r * 6, NtB);
            }
          }
        };
        if (i >= rlo) prefetch(i);
        for (; i >= rlo; --i) {
          const int cp0 = p0, cnb = nb, ccol = col, ccolB = colB;
          double cN[6], cNB[6];
#pragma unroll
          for (int q = 0; q < 6; ++q) { cN[q] = Nt[q]; cNB[q] = NtB[q]; }
          double xi[6];
          load_row6(xv + 6 * i, xi);   // final: every row above has been scattered (and the warp synchronised)
          if (i > rlo) prefetch(i - 1);
          // (a separator row also holds blocks of the other branch: columns outside [c0, c1) are skipped)
          const bool okA = ccol >= c0 && ccol < c1, okB = ccolB >= c0 && ccolB < c1;
          const double sdotA = (cN[0] * xi[0] + cN[1] * xi[1] + cN[2] * xi[2]) + (cN[3] * xi[3] + cN[4] * xi[4] + cN[5] * xi[5]);
          const double sdotB = (cNB[0] * xi[0] + cNB[1] * xi[1] + cNB[2] * xi[2]) + (cNB[3] * xi[3] + cNB[4] * xi[4] + cNB[5] * xi[5]);
          double* tA = xv + 6 * (okA ? ccol : 0) + r;
          double* tB = xv + 6 * (okB ? ccolB : 0) + r;
          const double vA = okA ? *tA : 0., vB = okB ? *tB : 0.;
          if (okA) *tA = vA - sdotA;
          if (okB) *tB = vB - sdotB;
          if (lane < 30)   // rows with more than ten blocks
            for (int a = g + 10; a < cnb; a += 5) {
              const int col2 = rcol[cp0 + a];
              if (col2 < c0 || col2 >= c1) continue;
              double N2[6];
              load_row6(b + (size_t)(cp0 - b0 + a) * 36 + r * 6, N2);
              const double sdot = (N2[0] * xi[0] + N2[1] * xi[1] + N2[2] * xi[2]) + (N2[3] * xi[3] + N2[4] * xi[4] + N2[5] * xi[5]);
              xv[6 * col2 + r] -= sdot;
            }
          __syncwarp();
        }
      } else if (pw >= 0) {
        if (k > 0) poses_of(k - 1);   // chunk k - 1 is done: x of its rows is final
        int lo, hi;                   // what the updates of chunk k read besides x, in flight during this chunk
        chunk_rows(k, lo, hi);
        const int i = first_row(lo);
        if (chunk_poses(k) && i < hi) pose_load(d, pt.cur, i, pin);
      }
      cp_async_wait_all();
      bar_sync(kBarBack, kSolveThreads);
    }
    if (pw >= 0 && nchunks > 0) poses_of(nchunks - 1);
    top = sChunk[nchunks];
    bar_sync(kBarBack, kSolveThreads);   // sChunk is rewritten by the next round
  }
}

// Between the forward and the backward pass the column-oriented index arrays in shared memory (upd_ptr, row_idx)
// are replaced by the row-oriented ones (rptr, rcol): entries [r0, r1) of rptr and [e0, e1) of rcol, in flight as one
// cp.async group.
__device__ void load_row_index(const BaDev& d, const SolveShared& S, int r0, int r1, int e0, int e1) {
  for (int i = r0 + (int)threadIdx.x; i < r1; i += kSolveThreads) cp_async4(S.upd_ptr + i, d.rptr + i);
  for (int i = e0 + (int)threadIdx.x; i < e1; i += kSolveThreads) cp_async4(S.row_idx + i, d.rcol + i);
  cp_async_commit();
}

// smem layout: [ring: cap*36 doubles][area: nsep*36 doubles][y: 6P doubles][meta ints: col_ptr (P+1),
//               upd_ptr (P+1), row_idx (nblk)][fixed-by-position bytes (P)]
// cap is a power of two >= 4 * (widest column of a branch + 1).
// kTimeline: the overlap timeline's instance (SVS_SOLVE_TIMING=3): the chain stamps each column it publishes
// kDiag: svs_chol6's marginals instance: the diagonal factor blocks are kept (factor_range)
template <bool kTimeline, bool kDiag>
__global__ void __launch_bounds__(kSolveThreads)
k_solve(BaDev d, int cap, int nsep, int refill_branch, int prof) {
  __shared__ int sFail[2][2];
  __shared__ double sRed[kSolveThreads / 32 + 2];
  __shared__ __align__(16) double sLbuf[2][2][28];
  __shared__ __align__(16) double sCdiag[22];
  __shared__ int sXfail;   // written by the other CTA of the cluster
  __shared__ int sChunk[kMaxChunks + 2];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int t = threadIdx.x, nt = kSolveThreads, lane = t & 31, warp = t >> 5;
  const int P = d.P, nblk = d.nblk;
  const int G = d.nbranch;                 // 1: a single chain, 2: two ends + separator (cluster of 2 CTAs)
  const int sep0 = d.branch_ptr[G];        // first separator column (= P when G == 1)
  const int my0 = d.branch_ptr[rank], my1 = d.branch_ptr[rank + 1];   // this CTA's branch
  const int sep_blk0 = G > 1 ? d.col_ptr[sep0] : nblk;
  SolveShared S;
  const int ring_off = 0, area_off = cap * 36;
  double* area = sm_solve + area_off;
  S.yv_off = area_off + nsep * 36;
  double* const yv_k = sm_solve + S.yv_off;
  int* meta = reinterpret_cast<int*>(yv_k + ((6 * (size_t)P + 1) / 2) * 2);
  S.col_ptr = meta; S.upd_ptr = S.col_ptr + (P + 1); S.row_idx = S.upd_ptr + (P + 1);
  S.sfix = reinterpret_cast<unsigned char*>(S.row_idx + nblk);
  S.fail = sFail; S.sL = sLbuf; S.cdiag = sCdiag;
  if (t < 4) sFail[t >> 1][t & 1] = 0;
  if (t == 4) sXfail = 0;
  if (t == 5) sRed[kSolveThreads / 32] = 0.;
  for (int i = t; i <= P; i += nt) { S.col_ptr[i] = d.col_ptr[i]; S.upd_ptr[i] = d.upd_ptr[i]; }
  for (int i = t; i < nblk; i += nt) S.row_idx[i] = d.row_idx[i];
  for (int i = t; i < P; i += nt) S.sfix[i] = d.fixed[d.perm[i]];
  const int p_first = t < P ? d.perm[t] : 0;   // the pose of this thread's first right-hand-side row
  const int rsep = d.rptr[sep0];               // row-major blocks of the rows before the separator
  // Everything above is the problem's structure, which no kernel of a trial writes, so it is staged before the wait.
  // In a chained trial every kernel executes pdl_wait() before pdl_launch_dependents(): the CTAs of this launch exist
  // only once k_build_wave is past its own wait, i.e. once everything enqueued before the build has completed (the
  // problem's set-up included).  What the build writes (S, bp, bc) and the control block (lambda, cur, the early exit)
  // are read below the wait.  Without programmatic serialisation (pdl == 0) the wait returns at once and the launch
  // itself follows the previous kernel.
  pdl_wait();
  pdl_launch_dependents();
  LmCtl* ctl = d.ctl;
  if (ctl->max_iters > 0 && (ctl->stop || ctl->iter >= ctl->max_iters)) return;   // speculatively enqueued trial: nothing left to do
  const unsigned long long t_start = global_ns();
  const long long c_start = clock64();
  if (rank == 0 && t == 0 && ctl->t_build_start) {   // the build before this launch has completed
    ctl->ns_build += (long long)(t_start - ctl->t_build_start);
    ctl->t_build_start = 0;
  }
  const double lambda = ctl->lambda;
  const int cur = ctl->cur;
  long long* const timeline = (kTimeline && d.dbg) ? d.dbg + 160 : nullptr;
  if (timeline && rank == 0 && t == 0) timeline[2 * d.P + 1] = (long long)global_ns();
  if (G > 1) {   // separator blocks: CTA 0 starts from S, CTA 1 from zero; both accumulate their branch's updates
    if (rank == 0) {
      for (int i = t; i < nsep * 18; i += nt) cp_async16(area + 2 * i, d.S + (size_t)sep_blk0 * 36 + 2 * i);
      cp_async_commit();
    } else {
      for (int i = t; i < nsep * 36; i += nt) area[i] = 0.;
    }
  }
  for (int j = t; j < P; j += nt) {   // right-hand side in elimination order: bs = bp - bc
    const bool mine = (j >= my0 && j < my1) || (rank == 0 && j >= sep0);
    const int p = j == t ? p_first : d.perm[j];
#pragma unroll
    for (int rr = 0; rr < 6; ++rr) yv_k[6 * j + rr] = mine ? d.bp[6 * p + rr] - d.bc[6 * p + rr] : 0.;
  }
  cp_async_wait_all();
  __syncthreads();
  long long tk[8];
  tk[0] = clock64();

  Team br;
  br.ring_off = ring_off; br.org = 0; br.mask = (unsigned)cap - 1u; br.cap = cap; br.prefilled = 0;
  br.j0 = my0; br.j1 = my1; br.sep_blk0 = sep_blk0; br.area_off = area_off; br.slot = 0; br.refill_period = refill_branch;
  br.prof = (prof == 2 && d.dbg) ? d.dbg + 12 + 16 * rank : nullptr;   // [.. + 32 + 3): unit phases of helper 0 (rank 0: dbg 44..46, rank 1: 56..58)
  br.timeline = timeline;
  factor_range<kTimeline, kDiag>(d, br, S, lambda);
  tk[1] = clock64();
  // In flight from here on: c = z on the branch rows, where the backward pass starts (the separator phase touches only
  // the separator rows of y), and the row-major index.  CTA 0 of two keeps the separator's part of the column-major one
  // until the separator is factored: rptr[0, sep0) and rcol[0, rptr[sep0]) lie below everything the separator's
  // columns read (upd_ptr[sep0, P], row_idx from col_ptr[sep0] on).
  for (int i = t; i < 3 * (my1 - my0); i += nt) cp_async16(yv_k + 6 * my0 + 2 * i, d.ywork + 6 * my0 + 2 * i);
  cp_async_commit();
  const bool split_index = G > 1 && rank == 0;
  load_row_index(d, S, 0, split_index ? sep0 : P + 1, 0, split_index ? rsep : nblk - P);
  int failed = sFail[0][0] | sFail[0][1];
  // The branch's backward pass walks the separator rows (x known, only scattered), then its own rows.  Its first round
  // is planned and its first chunk fetched before cluster sync #2 (plan_rows), where CTA 1 would otherwise idle.
  const Walk wb = G > 1 ? Walk{sep0, P, my0, my1} : Walk{my0, my1, 0, 0};
  if (G > 1) {
    if (rank == 1 && t == 0) sXfail = failed;   // read by CTA 0 below
    cluster.sync();   // #1: both branches factored, CTA 1's separator area and right-hand side complete
    tk[2] = clock64();
    if (rank == 0) {
      const double* rarea = cluster.map_shared_rank(area, 1);
      const double* ryv = cluster.map_shared_rank(yv_k, 1);
      const int* rfail = cluster.map_shared_rank(&sXfail, 1);
      for (int i = t; i < nsep * 18; i += nt) {
        const double2 a = reinterpret_cast<const double2*>(rarea)[i];
        double2* o = reinterpret_cast<double2*>(area) + i;
        const double2 b = *o;
        *o = make_double2(a.x + b.x, a.y + b.y);
      }
      for (int i = 6 * sep0 + t; i < 6 * P; i += nt) yv_k[i] += ryv[i];
      failed |= *rfail;
      __syncthreads();
      if (!failed) {
        Team sp;
        sp.ring_off = area_off; sp.org = sep_blk0; sp.mask = 0xffffffffu; sp.cap = nsep; sp.prefilled = 1;
        sp.j0 = sep0; sp.j1 = P; sp.sep_blk0 = nblk; sp.area_off = area_off; sp.slot = 1; sp.refill_period = 1 << 30; sp.prof = nullptr;
        sp.timeline = timeline;
        factor_range<kTimeline, kDiag>(d, sp, S, lambda);
        failed = sFail[1][0] | sFail[1][1];
      }
      tk[3] = clock64();
      load_row_index(d, S, sep0, P + 1, rsep, nblk - P);
      if (!failed) {   // the separator rows: c <- z, then solved
        for (int i = t; i < 3 * (P - sep0); i += nt) cp_async16(yv_k + 6 * sep0 + 2 * i, d.ywork + 6 * sep0 + 2 * i);
        cp_async_commit();
        cp_async_wait_all();
        __syncthreads();
        const PoseTail none = {false, false, 0., 0};
        double unused = 0.;
        scatter_rows(d, Walk{sep0, P, 0, 0}, sep0, P, ring_off, cap / 2, S, sChunk, false, none, unused);
        plan_rows(d, wb, wb.n(), ring_off, cap / 2, S, sChunk);
      }
      __syncthreads();
      // push the separator solution and the verdict into CTA 1
      double* rx = cluster.map_shared_rank(yv_k, 1);
      int* rf = cluster.map_shared_rank(&sXfail, 1);
      for (int i = 6 * sep0 + t; i < 6 * P; i += nt) rx[i] = yv_k[i];
      if (t == 0) *rf = failed;
    } else {
      cp_async_wait_all();
      __syncthreads();
      if (!failed) plan_rows(d, wb, wb.n(), ring_off, cap / 2, S, sChunk);
      tk[3] = tk[2];
    }
    cluster.sync();   // #2
    if (rank == 1) failed = sXfail;
  } else {
    cp_async_wait_all();
    __syncthreads();
    if (!failed) plan_rows(d, wb, wb.n(), ring_off, cap / 2, S, sChunk);
    tk[2] = tk[3] = tk[1];
  }
  tk[4] = clock64();
  if (failed) {
    cp_async_wait_all();
    if (rank == 0) {
      if (t == 0) { ctl->chol_fail = 1; ctl->scale_pose = 0; }
      for (int i = t; i < 7 * P; i += nt) d.pose[1 - cur][i] = d.pose[cur][i];
      for (int i = t; i < 12 * P; i += nt) d.Rt[1 - cur][i] = d.Rt[cur][i];
      for (int i = t; i < 6 * P; i += nt) d.x[i] = 0;
      if (t == 0) ctl->ns_solve += (long long)(global_ns() - t_start);
    }
    if (G > 1) cluster.sync();   // keeps the barrier count of the two CTAs equal (#3)
    return;
  }
  // --- backward pass of the branch with the pose update of its rows behind it (CTA 0 also updates the separator's
  //     poses): scale = sum x (lambda x + b)
  double sc = 0;
  const PoseTail poses = {G == 1 || rank == 0, true, lambda, cur};
  scatter_rows(d, wb, my0, my1, ring_off, cap / 2, S, sChunk, true, poses, sc);
  tk[5] = clock64();
  sc = warp_sum(sc);
  if (lane == 0) sRed[warp] = sc;
  __syncthreads();
  double total = 0;
  if (t == 0)
    for (int w = 0; w < nt / 32; ++w) total += sRed[w];
  if (G > 1) {
    if (rank == 1 && t == 0) *cluster.map_shared_rank(&sRed[kSolveThreads / 32], 0) = total;   // push into CTA 0
    cluster.sync();   // #3
  }
  if (rank == 0 && t == 0) {
    ctl->scale_pose = total + sRed[kSolveThreads / 32];
    ctl->chol_fail = 0;
    ctl->ns_solve += (long long)(global_ns() - t_start);
  }
  tk[6] = clock64();
  if (d.dbg && t == 0) {   // phase boundaries in cycles since the setup, and the setup itself from the wait on (slot 15
                           // of the CTA's role counters, which no role uses)
    for (int i = 1; i < 7; ++i) d.dbg[rank * 6 + i - 1] = tk[i] - tk[0];
    d.dbg[12 + 16 * rank + 15] = tk[0] - c_start;
  }
}

// ---------------------------------------------------------------------------------------- host side

namespace {
constexpr int kStaticSmem = 2048;   // static __shared__ of k_solve, rounded up
struct SolveDev { bool done = false; int smem_optin = 0; };
SolveDev g_dev[64];
std::mutex g_mu;

// per-device set-up (the attribute is per device; handles may live on several GPUs of one process)
int solve_smem_optin() {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return 0;
  std::lock_guard<std::mutex> lk(g_mu);
  SolveDev& s = g_dev[dev];
  if (!s.done) {
    cudaDeviceGetAttribute(&s.smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    cudaFuncSetAttribute(k_solve<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, s.smem_optin - kStaticSmem);
    cudaFuncSetAttribute(k_solve<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, s.smem_optin - kStaticSmem);
    cudaFuncSetAttribute(k_solve<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, s.smem_optin - kStaticSmem);
    s.done = true;
  }
  return s.smem_optin;
}

size_t solve_fixed_bytes(int P, int nblk, int nsep) {
  const size_t ybytes = (((size_t)6 * P * 8 + 15) / 16) * 16;
  const size_t mbytes = (((size_t)(2 * (P + 1) + nblk) * 4 + (size_t)P + 15) / 16) * 16;
  return ybytes + mbytes + (size_t)nsep * 288;
}
}  // namespace

// Shared-memory budget of k_solve: ring capacity (blocks, power of two) of one CTA for a problem whose
// separator columns hold nsep blocks (0 for a single chain); 0 if the fixed part alone does not fit.
int solve_ring_capacity(int P, int nblk, int nsep) {
  const int optin = solve_smem_optin();
  if (optin <= 0) return 0;
  const size_t budget = (size_t)optin - kStaticSmem - 256;
  const size_t fixed = solve_fixed_bytes(P, nblk, nsep);
  if (fixed >= budget) return 0;
  const int avail = (int)((budget - fixed) / 288);
  int cap = 1;
  while (cap * 2 <= avail) cap *= 2;
  return cap <= avail ? cap : 0;
}

// The chain/helper kernel runs when a CTA's ring holds 4 of its widest columns (it keeps two columns live and never
// checks residency on them); otherwise the global-memory kernel.
bool solve_uses_chain_kernel(const BaDev& d, int max_col_branch, int max_col_sep, int nsep) {
  const int G = d.nbranch;
  const int cap = d.P > 0 ? solve_ring_capacity(d.P, d.nblk, G > 1 ? nsep : 0) : 0;
  const int widest = G > 1 ? max_col_branch : max_col_sep;
  return !(cap == 0 || cap < 4 * (widest + 1) || cap / 2 < max_col_sep + 2 || G > 2);
}

// Launches k_solve, or the global-memory kernel (returns true).
bool launch_solve(const BaDev& d, int max_col_branch, int max_col_sep, int nsep, cudaStream_t st, int pdl, int keep_diag) {
  const int G = d.nbranch;
  if (!solve_uses_chain_kernel(d, max_col_branch, max_col_sep, nsep)) {
    launch_solve_general(d, st);
    return true;
  }
  int cap = solve_ring_capacity(d.P, d.nblk, G > 1 ? nsep : 0);
  const int widest = G > 1 ? max_col_branch : max_col_sep;
  while (G == 1 && cap / 2 >= d.nblk && cap / 2 >= 4 * (widest + 1)) cap /= 2;   // small problems: small ring
  int period = cap / (widest + 1) - 3;
  period = period < 1 ? 1 : (period > 64 ? 64 : period);
  const size_t smem = (size_t)cap * 288 + solve_fixed_bytes(d.P, d.nblk, G > 1 ? nsep : 0);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(G, 1, 1);
  cfg.blockDim = dim3(kSolveThreads, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = G; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 2 : 1;
  // 1: phase boundaries, 2: + per-role counters, 3: phase boundaries + the overlap timeline (when the chain publishes each
  // column; k_build_wave stamps when each column became complete)
  static const int prof = getenv("SVS_SOLVE_TIMING") ? std::max(1, atoi(getenv("SVS_SOLVE_TIMING"))) : 0;
  if (keep_diag) cudaLaunchKernelEx(&cfg, k_solve<false, true>, d, cap, G > 1 ? nsep : 0, period, prof);
  else if (prof >= 3) cudaLaunchKernelEx(&cfg, k_solve<true, false>, d, cap, G > 1 ? nsep : 0, period, prof);
  else cudaLaunchKernelEx(&cfg, k_solve<false, false>, d, cap, G > 1 ? nsep : 0, period, prof);
  return false;
}

}  // namespace svs
