// ba_types.cuh -- device-side view of one double-window BA problem.
// Layout follows what SlamGraph::copyDataToG2o (slam_graph.cpp:985-1032) hands to g2o,
// regrouped for the GPU: landmarks sorted by (anchor, pose set), edges grouped per landmark
// (self-anchor observation first), per-slot Hpl blocks in SoA.
#pragma once
#include <cuda_runtime.h>

namespace svs {

constexpr int kMaxIters = 64;
constexpr int kMaxTrack = 32;  // slots per landmark (anchor + observers) k_build stages in smem; longer tracks -> k_build_long

// Levenberg-Marquardt control block, lives in device memory; mirrors the locals of
// g2o::OptimizationAlgorithmLevenberg::solve (configured at slam_graph.cpp:336-346,1071-1073).
struct LmCtl {
  double lambda, ni;
  double chi_cur, chi_new, rho, scale_pose;
  int cur;         // index of the accepted state buffer
  int iter;        // outer iterations finished
  int qmax;        // trials in the running iteration
  int again;       // 1: run another trial of this iteration
  int stop;        // 1: Terminate (qmax == max_trials or rho == 0)
  int chol_fail;   // reduced system not positive definite in this trial
  int trials_total;
  int max_trials;
  int max_iters;   // > 0: kernels of trials enqueued past the end (or after Terminate) return at once
  // device durations of the trials of svs_ba_optimize's chained launch, where no stream event may sit between two kernels
  // (%globaltimer, ns): the first k_build_wave CTA past its wait -> k_solve past its wait; k_solve's CTA 0; the first
  // k_update CTA past its wait -> the end of its last CTA
  unsigned long long t_build_start, t_update_start;
  long long ns_build, ns_solve, ns_update;
  unsigned long long t_build0;   // overlap timeline (SVS_SOLVE_TIMING=3): %globaltimer at the entry of the first
                                 // k_build_wave CTA of the trial (0: none yet)
  double chi_init;
  double chi_iter[kMaxIters];
  double lambda_iter[kMaxIters];
  int trials_iter[kMaxIters];
};

struct BaDev {
  int P, L, E, C, nslots, nblk;   // E = internal edges = the caller's (E_user) + zero-weight padding edges (set_problem)
  int E_user;
  int flags;
  double f, px, py, b;
  // state, double buffered (index ctl->cur = accepted, the other = trial)
  double* pose[2];  // [P][7]
  double* Rt[2];    // [P][12]  row-major R, then t
  double* psi[2];   // [L][3]   internal landmark order
  const unsigned char* fixed;  // [P]
  // landmarks (internal order)
  const int* lm_eptr;            // [L+1]
  const int* lm_sptr;            // [L+1]
  const int* lm_anchor;          // [L]
  const unsigned char* lm_self;  // [L] first edge is the observation in the anchor frame
  const int* lm_user;            // [L] internal landmark -> the caller's landmark index
  // fused-kernel work lists: tasks = runs of landmarks with identical slot lists and <= 8 frames
  const int* task_lm;   // [ntasks] first landmark
  const int* task_cnt;  // [ntasks] landmarks in the task
  const int* gen_lm;    // [ngen] landmarks handled one warp each (9..32 slots, no observations)
  const int* long_lm;   // [nlong] landmarks with more than kMaxTrack slots (k_build_long)
  int ntasks, ngen, nlong;
  // edges (internal order)
  const int* e_pose;    // [E]
  const int* edge_src;  // internal edge -> index in the caller's arrays
  double* e_obs_w; double* e_w_w;   // writable views of e_obs / e_w (filled by k_regroup)
  const double* e_obs;  // [3][E]
  const double* e_w;    // [3][E] diagonal of Lambda
  // per-trial products of the fused kernel
  double* W;          // [18][nslots]  Hpl blocks (6x3 row-major), slot 0 of a landmark = anchor
  double* Dbl;        // [L][12]  Hll upper (d00 d01 d02 d11 d12 d22), b_l (3), pad
  double* chi_l;      // [L]  robust chi2 of the landmark's edges at the accepted state
  double* chi_new_l;  // [L]  ... at the trial state
  double* scale_l;    // [L]  sum dpsi (lambda dpsi + b_l)
  // reduced camera system
  double* S;       // [nblk][36] lower blocks in elimination order, pattern of the factor
  const int* tbl;  // [P*P] (block << 1 | transpose) for (row pose, col pose), -1 if absent
  double* bp;      // [6P] -J^T W e  (g2o _b, pose part)
  double* bc;      // [6P] Hpl Hll^-1 b_l
  double* x;       // [6P] pose increments, natural pose order
  // pose-pose constraints (G2oEdgeSE3)
  const int* c_i; const int* c_j; const double* c_T; const double* c_Lam;
  double* chi_c; double* chi_c_new;
  // factorisation structure (positions = elimination order)
  const int* perm; const int* pos;
  const int* col_ptr;  // [P+1] first block of column j is its diagonal block
  const int* row_idx;  // [nblk] row position of each block
  const int* upd_ptr;  // [P+1]
  const int* upd_dst;  // destination block of each (a>=b) pair of a column
  const int* upd_ab;   // (a << 16 | b): indices into the column's sub-diagonal list (b-major order)
  const int* urg_dst;  // [nblk] destination of pair (a, 0) of column j at col_ptr[j] + 1 + a
  double* Linv;        // [P][36] inverse of the diagonal factor blocks (general solver)
  const int* rptr;     // [P+1] row-major index of the off-diagonal factor blocks, columns descending inside a row
  const int* rowpos;   // [nblk] position of a block in that order (-1 for diagonal blocks)
  const int* rcol;     // [nblk - P] column of the block at a row-major position
  double* Nrow;        // [nblk - P][36] N_ij^T = (L_ij L_jj^-1)^T in row-major order, written by the forward pass of k_solve
  int nbranch;              // independent branches of the elimination tree (1 = a single chain)
  const int* branch_ptr;    // [nbranch + 1] column ranges of the branches; [nbranch] = first separator column
  double* ywork;       // [6P]
  double* part;        // [update grid][3] per-CTA partial sums (chi2 accepted, chi2 trial, scale)
  unsigned* ticket;    // [4] last-CTA-done counter of k_update; [1], [2]: task counter / warps-done counter of a persistent k_build_wave
  double* totals;      // [3] chi2 accepted / chi2 trial / scale of this rank's landmarks (sharded window)
  long long* dbg;      // [160 + 2P + 2] per-phase cycle counters of k_solve and k_build_wave; from 160 on the
                       // overlap timeline (SVS_SOLVE_TIMING=3): column ready, chain at column, build / solve entry
  // readiness of the block columns of S (elimination order), counted by k_build_wave on the overlap timeline runs
  const int* col_need;  // [P] work items that write column j or its right-hand side (build tasks + constraints)
  int* col_done;        // [P] of them finished in this trial (cleared by k_update)
  LmCtl* ctl;
};

}  // namespace svs
