// ba_kernels.cuh -- launchers of the BA kernels (ba_kernels.cu)
#pragma once
#include "ba_types.cuh"

namespace svs {
// true when kernel `slot` has not yet been given `bytes` of dynamic shared memory on the CURRENT device
// (cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device attribute); thread-safe
bool device_needs_smem_optin(int slot, size_t bytes);
size_t build_smem_bytes(int warps, int Kmax);
void launch_prep(const BaDev& d, int buf, cudaStream_t st);
void launch_regroup(const BaDev& d, const double* raw, cudaStream_t st);
void launch_build(const BaDev& d, int Kmax, int robust, double delta, cudaStream_t st);
// pdl = 1 (launch_build_wave, launch_solve, launch_update): launched with programmatic stream serialisation, so the
// kernel's CTAs are scheduled while the previous kernel of the stream still runs and wait for it on the device
// (svs_ba_optimize's trials, DESIGN.md 5)
// keep_diag = 1: k_solve also stores L_jj^-1 of every column into d.Linv (k_solve_general always does)
bool launch_solve(const BaDev& d, int max_col_branch, int max_col_sep, int nsep, cudaStream_t st, int pdl = 0,
                  int keep_diag = 0);   // true: k_solve_general
bool solve_uses_chain_kernel(const BaDev& d, int max_col_branch, int max_col_sep, int nsep);
void launch_build_wave(const BaDev& d, int robust, double delta, cudaStream_t st, int pdl = 0);
int solve_ring_capacity(int P, int nblk, int nsep);
void launch_solve_general(const BaDev& d, cudaStream_t st);
int update_grid_blocks(int L, int C);
void launch_update(const BaDev& d, int robust, double delta, int defer_decision, cudaStream_t st, int pdl = 0);
void launch_decide_deferred(const BaDev& d, cudaStream_t st);
void launch_chi2(const BaDev& d, int robust, double delta, cudaStream_t st);
void launch_export(const BaDev& d, double* out, cudaStream_t st);
// landmark blocks of (H + lambda I)^-1 into out [L][9] (caller's landmark order) from Z = S^-1 on the factor's pattern
// and the build's W / Dbl at the same lambda (ba_cov.cu)
void launch_point_cov(const BaDev& d, const double* Z, double lambda, double* out, cudaStream_t st);
// adjoint solve of svs_ba_observation_grad (ba_grad.cu): bp / bc of (H + lambda I) v = g from the build's W / Dbl, then,
// after the solve, v_l and dL/d(observations, weights) [E_user][3] in the caller's edge order (either may be nullptr)
void launch_grad_rhs(const BaDev& d, const double* g_pose, const double* g_psi, double lambda, cudaStream_t st);
// svs_ba_window_grad also: with cam_part (scratch [L][4]) the camera gradient into dcam [4], summed in a fixed order;
// nullptr launches the kernels svs_ba_observation_grad uses and nothing else
void launch_grad_edges(const BaDev& d, const double* g_psi, double lambda, int robust, double delta, double* dobs,
                       double* dinfo, double* cam_part, double* dcam, cudaStream_t st);
// after the solve: dL/d delta_c [C][6] and dL/dLambda_c [C][36] of every pose-pose constraint (either may be nullptr)
void launch_grad_constraints(const BaDev& d, double* dcT, double* dcLam, cudaStream_t st);
}  // namespace svs
