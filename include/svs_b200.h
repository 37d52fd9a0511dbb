/*
 * svs_b200.h -- C ABI of libsvsb200.so: H100-native (sm_90a) implementation of
 * ScaViSLAM's double-window bundle-adjustment iteration and dense stereo
 * front-end kernels.  Plain pointers and sizes only; no C++ or torch types.
 *
 * Every entry point names the reference interface it replaces
 * (paths relative to the ScaViSLAM tree, commit b29d070).
 *
 * Conventions
 *   SE3      double[7] = qx qy qz qw tx ty tz   (Eigen coeffs order; T_me_from_world)
 *   tangent  (upsilon, omega): translation first, left-multiplicative update
 *            T <- exp(delta) * T          (anchored_points.cpp:53-58)
 *   points   psi = (x/z, y/z, 1/z) in the anchor frame (maths_utils.h:66-69)
 *   status   0 = ok, <0 = error (svs_last_error gives the text); never throws
 *   threads  a handle may be used by one host thread at a time; distinct
 *            handles are independent (own stream, own workspaces)
 */
#ifndef SVS_B200_H
#define SVS_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define SVS_OK 0
#define SVS_ERR_INVALID (-1)      /* bad argument / index out of range */
#define SVS_ERR_CUDA (-2)         /* CUDA runtime error (text in svs_last_error) */
#define SVS_ERR_UNSUPPORTED (-3)  /* structurally valid input this build cannot take */
#define SVS_ERR_STATE (-4)        /* call order (e.g. optimize before set_problem) */
#define SVS_ERR_NOGPU (-5)        /* no CUDA device: there is NO CPU fallback */
#define SVS_ERR_NUMERIC (-6)      /* NaN residual (the reference throws std::runtime_error("Res is NaN!")) */

/* ------------------------------------------------------------------ BA */

typedef struct svs_ba svs_ba;

/* G2oCameraParameters (g2o_types/anchored_points.h:40-58) */
typedef struct {
  double f, px, py, b;
} svs_cam;

typedef struct {
  int device;        /* CUDA device ordinal, -1 = current device */
  int flags;         /* SVS_BA_* */
  int reserved[6];
} svs_ba_opts;

#define SVS_BA_DEFAULT 0
/* Skip the spurious J1'WJ1 prior g2o adds to the anchor pose for an observation
 * made in the landmark's own anchor frame (SURVEY.md B5).  Off = reference behaviour. */
#define SVS_BA_SKIP_SELF_ANCHOR_HESSIAN 1
/* Keep the pose ordering of the caller instead of the fill-reducing one. */
#define SVS_BA_NATURAL_ORDER 2

#define SVS_BA_MAX_ITERS 64

/* Mirrors g2o's per-iteration verbose line (slam_graph.cpp:1066) and
 * SlamGraph::Statistics (slam_graph.hpp:366-386). */
typedef struct {
  int iterations;                       /* return value of g2o optimize() */
  int trials_total;                     /* Levenberg trials (factorisations) */
  double chi2_init;
  double chi2_final;
  double lambda_final;
  double chi2_iter[SVS_BA_MAX_ITERS];   /* robust chi2 after outer iteration i */
  double lambda_iter[SVS_BA_MAX_ITERS];
  int trials_iter[SVS_BA_MAX_ITERS];
  int num_frames, num_points;           /* Statistics::num_frames / num_points */
  int num_point_edges, num_frame_edges; /* Statistics::num_point_edges / num_frame_edges */
  int nnzb_S;                           /* lower blocks of the reduced system incl. diagonal */
  int nnzb_L;                           /* blocks of its Cholesky factor */
  int max_track;                        /* longest landmark track (slots incl. anchor) */
  float ms_total;                       /* device time of the whole optimize() */
  float ms_build;                       /* fused linearise + Schur kernel, summed over trials */
  float ms_solve;                       /* reduced-system factor + solve + pose update */
  float ms_update;                      /* back-substitution + point update + trial chi2 */
  float ms_control;                     /* sharded window: the two all-reduces + LM decision kernel per trial */
  int launches;                         /* kernels launched by this call */
} svs_ba_stats;

/* Replaces: constructing g2o::SparseOptimizer + BlockSolver_6_3 + LinearSolverCSparse +
 * OptimizationAlgorithmLevenberg in SlamGraph::setupG2o (slam_graph.cpp:1063-1080). */
int svs_ba_create(const svs_ba_opts *opts, svs_ba **out);
void svs_ba_destroy(svs_ba *h);
const char *svs_last_error(const svs_ba *h);

/* Replaces SlamGraph::copyDataToG2o (slam_graph.cpp:985-1032) and the vertex/edge builders
 * addPoseToG2o / addPointToG2o / addObsToG2o / addConstraintToG2o
 * (slam_graph.cpp:907-920, slam_graph-impl.cpp:29-126).
 *   T_qt[P][7], fixed[P] (may be NULL = none fixed), psi[L][3]
 *   e_point/e_pose/e_anchor[E]: vertex 0/1/2 of each G2oEdgeProjectPSI2UVU as indices into the
 *     arrays above; all edges of a point must share one anchor (Point::anchorframe_id);
 *   e_obs[E][3] = (u, v, u_right); e_info_diag[E][3] = diagonal of Lambda
 *   c_i/c_j[C]: vertex 0/1 of each G2oEdgeSE3; c_T_ji[C][7] = measurement T_2_from_1;
 *   c_Lambda[C][36] row-major information.
 * Host buffers; copied to the device before the call returns.  Also performs the symbolic
 * analysis g2o does in BlockSolver::buildStructure + CSparse's symbolic phase. */
int svs_ba_set_problem(svs_ba *h, int P, const double *T_qt, const unsigned char *fixed,
                       int L, const double *psi,
                       int E, const int *e_point, const int *e_pose, const int *e_anchor,
                       const double *e_obs, const double *e_info_diag,
                       int C, const int *c_i, const int *c_j, const double *c_T_ji,
                       const double *c_Lambda, const svs_cam *cam);

/* svs_ba_set_problem for a window that already lies in GPU memory (assembled by CUDA code or held in
 * PyTorch tensors): the same arguments, but every array is a device pointer on the handle's device
 * (fixed may be NULL).  The structure analysis -- validation, grouping per landmark, the internal
 * landmark order, track padding, the build work lists and the co-visibility pattern -- runs on the
 * device; only a few counts and the P x P pattern (P*P/8 bytes) come back for the symbolic
 * factorisation.  Same return codes and svs_last_error texts as svs_ba_set_problem.
 *   A host pointer or memory of another device gives SVS_ERR_INVALID before anything is enqueued.
 *   The arrays are read on the handle's stream, which does not wait for other streams: the caller
 *   must have finished producing them (e.g. synchronised its own stream) before the call.  They may
 *   be reused or freed once the call returns.
 *   Calling it again with index arrays equal to the last device problem's re-sends only the numbers,
 *   device to device. */
int svs_ba_set_problem_device(svs_ba *h, int P, const double *T_qt, const unsigned char *fixed,
                              int L, const double *psi,
                              int E, const int *e_point, const int *e_pose, const int *e_anchor,
                              const double *e_obs, const double *e_info_diag,
                              int C, const int *c_i, const int *c_j, const double *c_T_ji,
                              const double *c_Lambda, const svs_cam *cam);

/* Replaces optimizer.initializeOptimization(); lm->setUserLambdaInit(lambda);
 * optimizer.optimize(num_iters) (slam_graph.cpp:336-346) with RobustKernelHuber(delta) on the
 * observation edges when `robust` (slam_graph-impl.cpp:86-90; the reference leaves delta = 1).
 * All iterations run on the device.  Returns g2o's value: iterations performed, -1 if the
 * problem is empty; <= -100 encodes an SVS_ERR_* as (-100 + err). */
int svs_ba_optimize(svs_ba *h, int num_iters, int robust, double huber_delta,
                    double lambda_init, int max_trials, svs_ba_stats *stats);

/* Replaces SlamGraph::restoreDataFromG2o (slam_graph.cpp:1037-1058); psi is returned in
 * inverse-depth form, xyz_anchor = invert_depth(psi). */
int svs_ba_get_poses(svs_ba *h, double *T_qt);
int svs_ba_get_points(svs_ba *h, double *psi);

/* Restore the state uploaded by set_problem (device-to-device; for repeated measurement). */
int svs_ba_reset_state(svs_ba *h);

/* SlamGraph::optimize(const OptParams&) in one call from host buffers
 * (north-star name; slam_graph.cpp:319-355): set_problem + optimize + get_*.
 * T_qt and psi are updated in place. */
int svs_optimiseInnerAndOuterWindow(svs_ba *h, int P, double *T_qt, const unsigned char *fixed,
                                    int L, double *psi,
                                    int E, const int *e_point, const int *e_pose, const int *e_anchor,
                                    const double *e_obs, const double *e_info_diag,
                                    int C, const int *c_i, const int *c_j, const double *c_T_ji,
                                    const double *c_Lambda, const svs_cam *cam,
                                    int num_iters, int robust, double huber_delta,
                                    svs_ba_stats *stats);

/* ---- one window split by landmarks across ranks (SURVEY.md 8e): every rank holds all poses, its
 * share of the landmarks and their edges; the reduced camera system is summed across ranks once per
 * Levenberg trial by the caller (ncclAllReduce / torch.distributed on the device buffers below), the
 * solve is replicated, back-substitution stays local.  Call order per trial:
 *   svs_ba_trial_build -> all-reduce(S, bp, bc) -> svs_ba_trial_solve -> all-reduce(totals) -> svs_ba_trial_decide */
/* Pose pairs that must be present in the block pattern of the reduced system although this rank
 * may hold no landmark coupling them (the whole window's pattern); call before svs_ba_set_problem.
 * A handle with a prescribed pattern adds no pose pairs of its own (its tracks with visibility drop-outs are
 * not completed with zero-weight edges), so that all handles of the window lay the system out identically;
 * npairs = 0 takes the prescription back. */
int svs_ba_set_structure(svs_ba *h, int npairs, const int *pose_i, const int *pose_j);
/* lm->setUserLambdaInit(lambda); ni = 2 (slam_graph.cpp:338-342) */
int svs_ba_lm_begin(svs_ba *h, double lambda_init, int max_trials);
int svs_ba_trial_build(svs_ba *h, int robust, double huber_delta);
/* Device pointers: S (nS doubles), bp and bc (nb doubles each), totals (3 doubles: chi2 at the
 * accepted state, chi2 at the trial state, sum dpsi (lambda dpsi + b_l) of this rank's landmarks). */
int svs_ba_system_buffers(svs_ba *h, double **S, long long *nS, double **bp, double **bc, long long *nb,
                          double **totals);
int svs_ba_trial_solve(svs_ba *h, int robust, double huber_delta);
int svs_ba_trial_decide(svs_ba *h, int *again, int *stop, int *iterations_done);
int svs_ba_lm_stats(svs_ba *h, svs_ba_stats *stats);

/* The same sharding driven INSIDE the library (one process per GPU): after svs_ba_comm_init the handle
 * owns an NCCL communicator, svs_ba_set_problem_sharded takes the WHOLE window on every rank and keeps
 * landmarks l with l % nranks == rank (poses replicated, pose-pose edges on rank 0, block pattern of the
 * whole window), and svs_ba_optimize runs every Levenberg trial as
 *   fused build -> ncclAllReduce(S | bp | bc, one packed buffer) -> replicated solve -> local
 *   back-substitution -> ncclAllReduce(3 scalars) -> identical decision on every rank
 * on the handle's stream without a host synchronisation in between (SlamGraph::optimize,
 * slam_graph.cpp:319-355, on a window too large for one GPU's latency budget).
 *   svs_comm_unique_id: rank 0 creates the 128-byte rendezvous id; the caller broadcasts it (MPI,
 *   torch.distributed, a socket).  NCCL is bound at run time (libnccl.so.2); SVS_ERR_STATE without it. */
int svs_comm_unique_id(char id[128]);
int svs_ba_comm_init(svs_ba *h, int nranks, int rank, const char id[128]);
int svs_ba_set_problem_sharded(svs_ba *h, int P, const double *T_qt, const unsigned char *fixed,
                               int L, const double *psi,
                               int E, const int *e_point, const int *e_pose, const int *e_anchor,
                               const double *e_obs, const double *e_info_diag,
                               int C, const int *c_i, const int *c_j, const double *c_T_ji,
                               const double *c_Lambda, const svs_cam *cam);
/* restoreDataFromG2o (slam_graph.cpp:1037-1058) for a sharded window: psi[L][3] of the WHOLE window on
 * every rank (svs_ba_get_points fills only this rank's landmarks of the same full-size array). */
int svs_ba_get_points_all(svs_ba *h, double *psi);

/* Inspection hooks used by the parity tests (device results copied to host buffers). */
/* g2o SparseOptimizer::activeRobustChi2 at the current state. */
int svs_ba_chi2(svs_ba *h, int robust, double huber_delta, double *chi2);
/* Reduced camera system the fused kernel produces at the current state:
 * S dense (6P x 6P row-major, symmetric, lambda included), bs (6P).  BlockSolver::solve
 * Schur part (g2o) on the system of BlockSolver::buildSystem. */
int svs_ba_reduced_system(svs_ba *h, int robust, double huber_delta, double lambda,
                          double *S_dense, double *bs, double *chi2);
/* Solve the reduced system once: x (6P) = S^-1 bs with the device block Cholesky
 * (LinearSolverCSparse::solve, slam_graph.cpp:55-60).  Returns 1 if not positive definite. */
int svs_ba_solve_reduced(svs_ba *h, int robust, double huber_delta, double lambda, double *x);

/* Marginal covariances of the window (g2o SparseOptimizer::computeMarginals for the caller who replaced all of
 * SlamGraph::optimize): blocks of (H + lambda I)^-1 over the free variables.
 *   State: the handle's accepted state -- the initial one after set_problem / set_problem_from_map, or the result of
 *     the last optimize.  H is the Gauss-Newton matrix the build kernels form there, with the robust weights of
 *     `robust` / `huber_delta` as in svs_ba_reduced_system; lambda (finite, >= 0) is added to every pose and landmark
 *     diagonal, as a Levenberg trial adds it.  The rows and columns of fixed poses are dropped (they are not
 *     variables): every block that involves a fixed pose is returned as zero.
 *   Outputs (each may be NULL; blocks row-major):
 *     pose_cov [P][36]       diagonal pose blocks in the caller's pose order, tangent order (upsilon, omega);
 *     pair_cov [npairs][36]  Cov(x_i, x_j) for i = pair_i[k], j = pair_j[k] (poses, any order; (j, i) is the transpose);
 *     point_cov [L][9]       landmark blocks in psi = (x/z, y/z, 1/z), the variable the optimiser estimates, in the
 *                            caller's landmark order; exactly symmetric; zero for a landmark without edges.  For
 *                            xyz_anchor = invert_depth(psi), apply the Jacobian J of invert_depth: J Sigma J^T.
 *   Method: one factor of the reduced system at lambda, one selected inversion on the factor's pattern (every pose
 *   pair a landmark couples lies in it), a solve of the block column of each requested pair outside the pattern, and
 *   Sigma_ll = D + sum_ab Y_a^T Z_ab Y_b per landmark (D = (Hll + lambda I)^-1, Y_a = Hpl_a D, Z = S^-1).
 *   Returns 0; 1 when the reduced system is not positive definite (all outputs zeroed); SVS_ERR_STATE before a problem
 *   is set; SVS_ERR_INVALID for lambda < 0 or not finite, npairs < 0, npairs > 0 with a null pair_i, pair_j or
 *   pair_cov, a pair index outside [0, P), and for lambda = 0 with no fixed pose (H is then exactly singular: every
 *   edge is invariant under one global SE3, SURVEY.md B2) -- all checked before anything is enqueued;
 *   SVS_ERR_UNSUPPORTED when the handle has a communicator (sharded windows).  The Levenberg state is left as it was
 *   found: a later svs_ba_optimize gives the same bits whether or not this call ran in between. */
typedef struct {
  int P, L, nnzb_L, nbranch, general;   /* as in svs_chol6_stats, for the handle's own factor */
  int n_pairs_in_pattern;               /* pairs served from the selected inversion */
  int n_cols_solved;                    /* block columns solved for pairs outside the factor's pattern */
  float ms;                             /* device time: build + factor + inversion + landmark kernel */
} svs_ba_cov_stats;
int svs_ba_covariance(svs_ba *h, int robust, double huber_delta, double lambda, double *pose_cov, int npairs,
                      const int *pair_i, const int *pair_j, double *pair_cov, double *point_cov,
                      svs_ba_cov_stats *stats);

/* Gradient of a loss of the optimised window with respect to its observations and their weights (the adjoint of the
 * minimiser), for a caller who trains observations or confidence weights through the back-end.
 *   State: the handle's accepted state x*, which must be a stationary point of the cost: optimise to convergence first.
 *   Notation: e_e = z_e - h_e(x) the stereo residual of edge e and J_e = de_e/dx; Omega_e = diag(e_info[e]); rho'_e the
 *     Huber weight at x* when `robust` (huber_delta), else 1; the pose tangent is delta = (upsilon, omega) of
 *     T <- exp(delta) T, psi is updated additively.  H = sum_e rho'_e J_e^T Omega_e J_e + the pose-pose blocks.
 *   Given g = (dL/d delta_p, dL/d psi_l):  (H + lambda I) v = g over the free variables (fixed poses and landmarks
 *     without edges are not variables, their v is 0), then per caller edge
 *       dL_dobs[e]  = -rho'_e Omega_e (J_e v),      dL_dinfo[e][k] = -rho'_e e_{e,k} (J_e v)_k.
 *   Conditions:
 *   - rho'_e is held at its value at x*: no rho'' or residual-curvature terms.  This is the exact derivative of the
 *     minimiser when the residuals vanish and its Gauss-Newton approximation otherwise.
 *   - H never contains the self-anchor term of SURVEY.md B5, whatever the handle's flags (that term is not a derivative
 *     of the cost: J_pose = -J_anchor when pose == anchor).  This is where the result deliberately differs from the H of
 *     svs_ba_covariance.
 *   - Not differentiated here: the pose-pose constraints (they enter H, but get no gradient), the camera, the initial
 *     state.  svs_ba_window_grad below adds the constraints and the camera.
 *   - An edge whose three weights are all 0 gets 0 in both outputs; the zero-weight padding edges the library adds
 *     produce nothing.  For a window from svs_ba_set_problem_from_map the caller's edge order is svs_map_last_edges'.
 *   Arrays: dL_dpose [P][6] (upsilon, omega) and dL_dpsi [L][3] in the caller's orders, NULL = 0; dL_dobs, dL_dinfo
 *   [E][3] in the caller's edge order, each may be NULL.  on_device != 0: all four are device pointers on the handle's
 *   device, ready when the call is made.  The call returns after the outputs have been written.
 *   Method: one build at x* and lambda, one factor and solve of the reduced system, and two light kernels.
 *   Returns 0; 1 when the reduced system is not positive definite (outputs zeroed); SVS_ERR_STATE before a problem is
 *   set; SVS_ERR_INVALID for lambda < 0 or not finite, lambda = 0 with no fixed pose (H is exactly singular, SURVEY.md
 *   B2) and, with on_device, an array that is not memory of the handle's device -- all checked before anything is
 *   enqueued; SVS_ERR_UNSUPPORTED when the handle has a communicator (sharded windows).  The Levenberg state is left
 *   as it was found. */
typedef struct {
  int P, L, E, nnzb_L, nbranch, general;   /* as svs_ba_cov_stats; E = the caller's edges */
  float ms;                                /* device time: build + factor + solve + adjoint kernels */
} svs_ba_grad_stats;
int svs_ba_observation_grad(svs_ba *h, int robust, double huber_delta, double lambda, const double *dL_dpose,
                            const double *dL_dpsi, double *dL_dobs, double *dL_dinfo, int on_device,
                            svs_ba_grad_stats *stats);

/* svs_ba_observation_grad extended to the pose-pose constraints and the stereo camera, from the same v (one build, one
 * factor, one solve; State, Notation and Conditions as above, except that the constraints and the camera are now
 * differentiated), for a caller who learns constraint information, constraint measurements or the calibration.
 *   Pose-pose constraint c (G2oEdgeSE3, i = c_i[c], j = c_j[c]): e_c = log(T_ji T_i T_j^-1), cost e_c^T Lambda_c e_c,
 *     J_i = third(T_ji, e_c), J_j = -third(I, -e_c) (anchored_points.cpp:207-215; zero for a fixed pose) and
 *     w_c = J_i v_i + J_j v_j.  Then
 *       dL_dcLambda[c][a][b] = -(w_{c,a} e_{c,b} + w_{c,b} e_{c,a}) / 2   the gradient of each entry as the cost uses
 *                                                                        it (symmetric; on the diagonal the form of
 *                                                                        dL_dinfo)
 *       dL_dcT[c]            = -X_c^T Lambda_c w_c,  X_c = third(I, e_c)  in the tangent (upsilon, omega) of
 *                                                                        T_ji <- exp(delta) T_ji
 *     A constraint whose two poses are fixed gets exactly 0.  Every row of the caller's constraint arrays is its own
 *     input (the reference adds each pair in both orders, SURVEY.md B4).
 *   Camera (svs_cam): e_e is linear in z_e, so dL_dcam[k] = sum_e (de_e/dcam_k)^T dL_dobs[e] with y the point in the
 *     observing camera: de/df = -(y0, y1, y0 - b) / y2, de/dpx = -(1, 0, 1), de/dpy = -(0, 1, 0), de/db = (0, 0, f / y2).
 *     Self-anchored edges count (their J v is the psi block alone); edges with all-zero weights add nothing.  The sum
 *     runs in a fixed order without atomics: the same bits on every call.
 *   Like dL_dinfo, dL_dcLambda and dL_dcT are first order in the residual where the residuals do not vanish.
 *   Arrays: as svs_ba_observation_grad, the outputs in *out (out or any member may be NULL: that output is neither
 *   computed nor written).  dL_dcT [C][6] and dL_dcLambda [C][36] (row-major) are in the caller's constraint order --
 *   for a window from svs_ba_set_problem_from_map, the order of the arrays passed to it; dL_dcam [4] is (f, px, py, b).
 *   Returns: as svs_ba_observation_grad (1: every requested output zeroed), with the same checks in the same order.
 *   Not differentiated: fixed-pose values and the initial state (zero at a stationary point); sharded windows give
 *   SVS_ERR_UNSUPPORTED. */
typedef struct {
  double *dL_dobs, *dL_dinfo; /* [E][3], the caller's edge order (as svs_ba_observation_grad) */
  double *dL_dcT;             /* [C][6]  tangent (upsilon, omega) of T_ji <- exp(d) T_ji, the caller's constraint order */
  double *dL_dcLambda;        /* [C][36] row-major, symmetric */
  double *dL_dcam;            /* [4]     f, px, py, b */
} svs_ba_grad_out;            /* any member may be NULL */
int svs_ba_window_grad(svs_ba *h, int robust, double huber_delta, double lambda, const double *dL_dpose,
                       const double *dL_dpsi, const svs_ba_grad_out *out, int on_device, svs_ba_grad_stats *stats);

/* ------------------------------------------------------------------ block Cholesky of a caller's 6x6-block system
 * g2o::LinearSolver<Matrix6d>::solve(A, x, b) as LinearSolverCSparse implements it (slam_graph.cpp:55-60), for a
 * caller that keeps g2o and hands its reduced camera system to the device (INTEGRATION.md).  The elimination order,
 * the two-ended split and the choice between the cluster solver and the global-memory solver are those of the BA
 * handle above; a handle owns one internal svs_ba for them.
 *
 * Input: the upper triangle of a symmetric positive-definite matrix in block CCS, as g2o's
 * SparseBlockMatrix::fillCCS(..., upperTriangle = true) sees it:
 *   col_ptr[P + 1]   starts at 0 and never decreases; nnzb = col_ptr[P];
 *   row_idx[nnzb]    strictly ascending within each column, row <= column; every column has its diagonal block;
 *   blocks[nnzb][36] each block column-major (Eigen's Matrix6d::data()).
 * Only the upper triangle of a diagonal block is read (its lower triangle may hold anything), as CSparse reads an
 * upper-triangular input.  b and x hold 6P entries in the caller's block order.  The damping is already on the
 * diagonal (g2o's Levenberg adds lambda before it calls the linear solver): nothing is added or fixed here.
 * on_device != 0: blocks, b and x are device pointers on the handle's device (e.g. torch CUDA tensors), ready when
 * the call is made; the pattern arrays are always host arrays (the symbolic analysis runs on the host).
 * The call returns after x has been written.
 *
 * Returns 0 solved; 1 not positive definite (g2o's solve returns false and the trial is rejected), x is zeroed;
 * SVS_ERR_INVALID for a malformed pattern or a null pointer, checked before anything is enqueued (the handle stays
 * usable); SVS_ERR_CUDA for a device error.  svs_chol6_create returns SVS_ERR_NOGPU without a device: there is no CPU
 * fallback.  One handle per thread; each handle has its own stream.
 *
 * The symbolic analysis is cached: a call whose pattern equals the previous call's (a cheap host comparison of
 * col_ptr and row_idx) reuses it, as do the trials of one g2o optimize().  svs_chol6_init is LinearSolver::init():
 * it forgets the cached analysis. */
typedef struct svs_chol6 svs_chol6;
typedef struct {
  int P, nnzb_A, nnzb_L;   /* block columns, upper blocks given, blocks of the factor */
  int nbranch;             /* 2 = two-ended elimination, 1 = one chain */
  int general;             /* 1 = k_solve_general ran */
  int symbolic_reused;     /* 1 = the cached analysis of the same pattern was used */
  float ms;                /* device time of scatter + factor + solve */
} svs_chol6_stats;
int svs_chol6_create(int device, svs_chol6 **out);   /* device < 0: the current device */
void svs_chol6_destroy(svs_chol6 *h);
const char *svs_chol6_last_error(const svs_chol6 *h);
int svs_chol6_init(svs_chol6 *h);
int svs_chol6_solve(svs_chol6 *h, int P, const int *col_ptr, const int *row_idx, const double *blocks,
                    const double *b, double *x, int on_device, svs_chol6_stats *stats);

/* Marginals: blocks of A^-1 from the same factor, as LinearSolverCSparse's solveBlocks / solvePattern compute them
 * for SparseOptimizer::computeMarginals.  The pattern, blocks, on_device, the return codes, the validation and the
 * analysis cache are those of svs_chol6_solve (a solve and an inversion on one pattern share one analysis).  Every
 * block the factor stores (the pattern of A plus fill-in) comes from one selected inversion over the factor; a
 * requested block outside it from a solve of its block column (stats->n_cols_solved).  Each output block is
 * column-major (Eigen's data()); block (r, c) with r > c is the transpose of (c, r), so any order is valid.
 * Returns 1 with all outputs zeroed when A is not positive definite.  req_r / req_c are always host arrays; a request
 * outside [0, P), n < 0 or a null request array with n > 0 is SVS_ERR_INVALID, before anything is enqueued. */
typedef struct {
  int P, nnzb_A, nnzb_L, nbranch, general, symbolic_reused;   /* as in svs_chol6_stats */
  int n_in_pattern;        /* requests served from the selected inversion */
  int n_cols_solved;       /* block columns solved for requests outside the factor's pattern */
  float ms;                /* device time of scatter + factor + inversion */
} svs_chol6_inv_stats;
/* LinearSolver::solveBlocks(blocks, A): the P diagonal blocks of A^-1, inv_diag [P][36] column-major */
int svs_chol6_solve_blocks(svs_chol6 *h, int P, const int *col_ptr, const int *row_idx, const double *blocks,
                           double *inv_diag, int on_device, svs_chol6_inv_stats *stats);
/* LinearSolver::solvePattern(spinv, blockIndices, A): blocks (req_r[k], req_c[k]) of A^-1, out [n][36] column-major */
int svs_chol6_solve_pattern(svs_chol6 *h, int P, const int *col_ptr, const int *row_idx, const double *blocks,
                            int n, const int *req_r, const int *req_c, double *out, int on_device,
                            svs_chol6_inv_stats *stats);

/* ------------------------------------------------------------------ FAST grid detector */

typedef struct svs_fast svs_fast;

/* FastGridCell (keyframes.h:30-43): cv::Range urange [u0,u1), vrange [v0,v1), fast_thr */
typedef struct {
  int u0, u1, v0, v1, thr;
} svs_fast_cell;

/* Private members of FastGrid (fast_grid.h:52-63) */
typedef struct {
  int grid_w, grid_h, fast_min, fast_max;
  int min_inner, min_outer, max_inner, max_outer;
} svs_fast_grid_params;

int svs_fast_create(int device, int max_w, int max_h, int max_keypoints, svs_fast **out);
void svs_fast_destroy(svs_fast *h);
const char *svs_fast_last_error(const svs_fast *h);

/* FastGrid::FastGrid (fast_grid.cpp:23-58): fills the band limits and grid_w*grid_h cells. */
int svs_fast_grid_init(int img_w, int img_h, int num_features_per_cell, int boundary_per_cell, int fast_thr,
                       int grid_w, int grid_h, int fast_min, int fast_max, svs_fast_grid_params *grid,
                       svs_fast_cell *cells);

/* The uint8 pyramid level the detector runs on (cv::Mat img of FastGrid::detect*).  Host buffer
 * (copied H2D) or a device buffer already resident (copied D2D into the handle's pitched image). */
int svs_fast_set_image(svs_fast *h, const unsigned char *img, int pitch, int w, int height);
int svs_fast_set_image_device(svs_fast *h, const unsigned char *d_img, int pitch, int w, int height);

/* FastGrid::detect (fast_grid.cpp:60-83): cv::FastFeatureDetector(cell.thr, false) on every cell
 * ROI.  out_xy[n][2] = (x + u0, y + v0) grouped by cell in list order, raster order inside a cell,
 * so the reference's quadtree content (index within the cell) is i - cell_off[c].
 * cell_off[ncells + 1].  Returns the total number of keypoints (may exceed max_out; only
 * max_out are written) or a negative SVS_ERR_*. */
int svs_fast_detect(svs_fast *h, const svs_fast_cell *cells, int ncells, int *out_xy, int max_out, int *cell_off);

/* FastGrid::detectAdaptively (fast_grid.cpp:86-152): up to `trials` re-detections per cell with
 * the threshold walk of the reference (state shared along a grid row); cells[].thr is updated in
 * place like FastGrid::cell_grid2d_. */
int svs_fast_detect_adaptively(svs_fast *h, const svs_fast_grid_params *grid, svs_fast_cell *cells, int trials,
                               int *out_xy, int max_out, int *cell_off);

/* ------------------------------------------------------------------ dense photometric tracker */

typedef struct svs_dt svs_dt;

#define SVS_DT_MAX_LEVELS 8
/* Bilinear taps with exact float weights instead of the texture unit's 8-fractional-bit weights
 * (the reference binds the images as linearly filtered textures, gpu/dense_tracking.cu:285-287). */
#define SVS_DT_EXACT_BILINEAR 1

typedef struct {
  double chi2[SVS_DT_MAX_LEVELS];   /* final photometric chi2 per level */
  int passes[SVS_DT_MAX_LEVELS];    /* fused (chi2 + J^T J + J^T r) pixel passes per level */
  int launches;
  float ms_total;
} svs_dt_stats;

/* Replaces GpuTracker::GpuTracker (gpu/dense_tracking.cu:265-299) + the GpuMat members of
 * DenseTracker / FrameData: device images for `nlevels` pyramid levels of a w0 x h0 frame. */
int svs_dt_create(int device, int w0, int h0, int nlevels, int flags, svs_dt **out);
void svs_dt_destroy(svs_dt *h);
const char *svs_dt_last_error(const svs_dt *h);

/* GpuIntrinsics::set (gpu/dense_tracking.cuh:28-41) of level l (cam_vec[l], dense_tracking.cpp:82-84) */
int svs_dt_set_intrinsics(svs_dt *h, int level, float focal_length, float px, float py);
/* The float images GpuTracker::bindTexture / jacobianReduction take (dense_tracking.cpp:88-104):
 * previous-frame intensity, current intensity and its x/y derivatives; host buffers with
 * `stride_floats` floats per row; NULL keeps the resident plane. */
int svs_dt_set_images(svs_dt *h, int level, const float *prev, const float *cur, const float *dx,
                      const float *dy, int stride_floats);
/* frame_data_.gpu_disp_32f (level-0 disparity) for computePointCloud */
int svs_dt_set_disparity(svs_dt *h, const float *disp, int stride_floats, int w, int height);
/* DenseTracker::computeDensePointCloudGpu (dense_tracking.cpp:195-216): cams[nlevels] are the
 * per-level StereoCamera parameters (frame_grabber-impl.cpp:50-59). */
int svs_dt_compute_point_cloud(svs_dt *h, const double T_cur_from_actkey[7], const svs_cam *cams);
/* dev_ref_dense_points_[level] as packed float4 (w*h*4 floats) */
int svs_dt_set_point_cloud(svs_dt *h, int level, const float *cloud_xyzw);
int svs_dt_get_point_cloud(svs_dt *h, int level, float *cloud_xyzw);
/* GpuTracker::chi2 (gpu/dense_tracking.cu:455-491) */
int svs_dt_chi2(svs_dt *h, int level, const double T_cur_from_prev[7], double *chi2);
/* GpuTracker::jacobianReduction (gpu/dense_tracking.cu:318-356): Hessian in GpuSymMatrix6 packing
 * (21 values: for r: for c <= r), jacobian_times_res (6) */
int svs_dt_jacobian_reduction(svs_dt *h, int level, const double T_cur_from_prev[7], double H21[21],
                              double b6[6], double *chi2);
/* GpuTracker::residualImage (gpu/dense_tracking.cu:494-567; called once per level at the end of
 * denseTrackingGpu, dense_tracking.cpp:180-188): res_rgba = w*h packed float4 -- grey max(0, 1 - 50 r^2) where the
 * pixel contributes, (1,0,0,1) where it projects outside the frame, (0,1,0,1) where it has no depth */
int svs_dt_residual_image(svs_dt *h, int level, const double T_cur_from_prev[7], float *res_rgba);
/* DenseTracker::denseTrackingGpu (dense_tracking.cpp:62-193): coarse-to-fine LM, T updated in place */
int svs_dt_track(svs_dt *h, double T_cur_from_actkey[7], svs_dt_stats *stats);

/* ---- the tracker the reference builds WITHOUT SCAVISLAM_CUDA_SUPPORT (SURVEY.md 8 row a18):
 * DenseTracker::denseTrackingCpu / computeDensePointCloudCpu (dense_tracking.cpp:222-423): every 4th pixel,
 * previous intensity from the uint8 pyramid, residual clamped to +-0.1, exact software bilinear taps, FP64
 * point transform, border test isInFrame(uv, 2), disparity scaled by 2^-level, H not damped.  Level sizes
 * must be multiples of 4 (the reference asserts the same).  Pixel sums are FP64 (reference: sequential FP32). */
typedef struct svs_dtc svs_dtc;
int svs_dtc_create(int device, int w0, int h0, int nlevels, svs_dtc **out);
void svs_dtc_destroy(svs_dtc *h);
const char *svs_dtc_last_error(const svs_dtc *h);
/* frame_data_.prev_left().pyr_uint8[level]; on_device != 0: img is a device pointer (e.g. svs_prep_level) */
int svs_dtc_set_prev_u8(svs_dtc *h, int level, const unsigned char *img, int pitch, int on_device);
/* frame_data_.pyr_float32 / pyr_float32_dx / pyr_float32_dy [level]; NULL planes are left as they are */
int svs_dtc_set_cur(svs_dtc *h, int level, const float *cur, const float *dx, const float *dy, int stride_floats,
                    int on_device);
/* frame_data_.disp (level-0 float disparity, host) */
int svs_dtc_set_disparity(svs_dtc *h, const float *disp, int stride_floats);
/* computeDensePointCloudCpu(T_cur_from_actkey) with cam_vec[level] = cams[level] */
int svs_computeDensePointCloudCpu(svs_dtc *h, const double T_cur_from_actkey[7], const svs_cam *cams);
/* ref_dense_points_[level]: (h/4) x (w/4) float4, tightly packed */
int svs_dtc_get_point_cloud(svs_dtc *h, int level, float *cloud_xyzw);
int svs_dtc_set_point_cloud(svs_dtc *h, int level, const float *cloud_xyzw);
/* denseTrackingCpu(&T_cur_from_actkey): coarse-to-fine, T updated in place */
int svs_denseTrackingCpu(svs_dtc *h, const svs_cam *cams, double T_cur_from_actkey[7], svs_dt_stats *stats);

/* ------------------------------------------------------------------ guided patch matcher */

typedef struct svs_matcher svs_matcher;
#define SVS_MATCH_MAX_LEVELS 4

/* cam_vec[level] (LinearCamera part of StereoCamera): image size, focal length, principal point */
typedef struct {
  int w, h;
  double f, px, py;
} svs_match_level;

/* CandidatePoint<3> (data_structures.h): anchor keyframe (slot given to svs_matcher_set_keyframe,
 * -1 = not in vertex_map), xyz in the anchor frame, its (u, v) observation at anchor_level */
typedef struct {
  int keyframe;
  int anchor_level;
  double xyz_anchor[3];
  double anchor_obs_pyr[2];
} svs_match_point;

/* One entry per candidate point, in input order.  matched == 1 entries, in order, are what the
 * reference appends to TrackData::obs_list / point_list / ba2globalptr. */
typedef struct {
  int predicted;       /* computePrediction succeeded */
  int textured;        /* key patch passed the thr_std test */
  int matched;         /* a candidate beat thr_mean and the disparity is valid */
  int n_candidates;    /* FAST corners inside the search window */
  int index;           /* quadtree content of the best candidate, -1 = none */
  int min_dist;        /* its score (literal formula of matcher.cpp:73) */
  int uv_pyr[2];       /* its position at anchor_level */
  double obs[3];       /* (u, v, u_right) at level 0 */
  double xyz_actkey[3];
} svs_match_result;

int svs_matcher_create(int device, int nlevels, const svs_match_level *levels, int max_keyframes, int max_points,
                     int max_keypoints, svs_matcher **out);
void svs_matcher_destroy(svs_matcher *h);
const char *svs_matcher_last_error(const svs_matcher *h);
/* keyframe_map[id].pyr + vertex_map[id].T_me_from_w for one anchor keyframe (uint8 pyramid, host) */
int svs_matcher_set_keyframe(svs_matcher *h, int slot, const double T_me_from_w[7], const unsigned char *const *pyr,
                           const int *pitch);
/* cur_frame.pyr + cur_frame.disp (level-0 float disparity); either may be NULL to keep what is loaded */
int svs_matcher_set_current(svs_matcher *h, const unsigned char *const *pyr, const int *pitch, const float *disp,
                          int disp_pitch_floats);
/* feature_tree.at(level): the FAST corners (x, y) and their quadtree content (index within the cell) */
int svs_matcher_set_features(svs_matcher *h, int level, const int *xy, const int *content, int n);
/* The same from the FAST handle's last svs_fast_detect* result where it lies on the device (content = ordinal of the
 * corner inside its cell, fast_grid.cpp:75-80): the corners never travel through host memory. */
int svs_matcher_set_features_from_fast(svs_matcher *h, int level, svs_fast *fast);
/* GuidedMatcher<StereoCamera>::match (matcher.cpp:312-398).  T_actkey_from_w replaces
 * vertex_map[actkey_id].  Returns the number of matched points or a negative SVS_ERR_*. */
int svs_match(svs_matcher *h, const double T_cur_from_actkey[7], const double T_actkey_from_w[7],
              const svs_match_point *pts, int n, int search_radius, int thr_mean, int thr_std,
              svs_match_result *out);

/* ------------------------------------------------------------------ the tracked frame's bookkeeping
 * StereoFrontend::processFrame after the LM (stereo_frontend.cpp:184-306): matchAndTrack's candidate groups and budget
 * (:977-1065), processMatchedPoints (:834-974), shallWeDropNewKeyframe (:512-528) and addMorePointsToOtherFrame
 * (:724-823, the seeding of addNewPoints and addNewKeyframe).  Everything is read from the matcher handle: the results
 * and candidates of its last match, the current frame's FAST corners per level and its level-0 disparity. */

/* the reference's ui / params_ values; SVS_FRONTEND_PARAMS_DEFAULT mirrors them */
typedef struct {
  unsigned long long seed;     /* emission order of the seeding (see svs_addMorePoints) */
  float max_reproj_error;      /* ui.max_reproj_error */
  int newpoint_clearance;      /* params_.newpoint_clearance, R in [0, 64] */
  int num_max_points;          /* ui.num_max_points: the seeding keeps at most (num_max_points >> l) + 1 points at
                                  level l (matchAndTrack's budget is an argument of svs_match_track) */
  int min_num_points;          /* ui.min_num_points: add flag (i, j) = grid3x3[i][j] <= min_num_points */
  int featureless_corners_thr; /* params_.new_keyframe_featuerless_corners_thr */
  float parallax_thr;          /* ui.parallax_thr */
} svs_frontend_params;
#define SVS_FRONTEND_PARAMS_DEFAULT {0ull, 2.f, 2, 300, 25, 2, 0.75f}

/* PointStatistics (stereo_frontend.h:160-177) and av_track_length_.  Grid index i comes from u, j from v:
 * grid2x2[i][j] with i = 0 when u < (int)(w * 0.5); grid3x3[i][j] with the thirds (int)(w * third) and
 * (int)(w * 2 * third), float third = 1./3. (w, h of matcher level 0). */
typedef struct {
  int num_matched_points[SVS_MATCH_MAX_LEVELS];
  int grid2x2[2][2];
  int grid3x3[3][3];
  double av_track_length;   /* sum of ||uv_pyr - curkey_uv_pyr|| in match order (double) / num_tracked: NaN at 0 */
  int num_tracked;          /* entries that passed the gate */
  int num_new;              /* of which new two-view points */
} svs_point_stats;

/* one gated match, in match order: candidate index, class (1 = NewTwoViewPoint, index < n_new; 0 = TrackPoint),
 * anchor level and the observation uvu at level 0 */
typedef struct {
  int index;
  int is_new;
  int anchor_level;
  int reserved;
  double uvu[3];
} svs_tracked_point;

/* one seeded CandidatePoint<3>: level, uv_pyr, uvu_pyr = (u, v, u - disp), xyz = T_newkey_from_cur * xyz_cur and
 * normal = -xyz_cur / |xyz_cur| (xyz_cur = unmap_uvu(uvu_pyr * 2^level), the normal is not transformed) */
typedef struct {
  int level;
  int reserved;
  double uv_pyr[2];
  double uvu_pyr[3];
  double xyz[3];
  double normal[3];
} svs_new_point;

/* matchAndTrack's matching (stereo_frontend.cpp:977-1065) in one call.  The n candidates come as n_groups >= 2
 * consecutive groups ending at group_end[g] (non-decreasing, group_end[n_groups-1] = n): group 0 is
 * newpoint_map[actkey], groups 1 .. n_groups-2 the neighbours' newpoint_map lists in the order the caller walks
 * strength_to_neighbors (weakest first), the last group the neighbourhood's point_list.  One k_match launch covers all
 * candidates (an entry does not depend on the others, so matching groups that are then discarded is exact); a device
 * kernel then applies the stop rule: neighbour group g is kept iff 2 * (matched entries of groups 0 .. g-1) <
 * num_max_points and every earlier neighbour group was kept.  Entries of a group that is not kept get matched = 0; their
 * other fields mean nothing.  The device results are then the reference's TrackData in order, and
 * svs_calcFastMotionOnly_matched / svs_processMatchedPoints work on them as after svs_match.  *num_new_feat_matched =
 * matched entries of groups 0 .. n_groups-2 (the new-point boundary in candidate order is group_end[n_groups-2]),
 * *num_obs = all matched entries.  out (n entries) may be NULL.  Returns SVS_OK or a negative SVS_ERR_*; a refused
 * call leaves the results of the previous match in place. */
int svs_match_track(svs_matcher *h, const double T_cur_from_actkey[7], const double T_actkey_from_w[7],
                    const svs_match_point *pts, int n, int n_groups, const int *group_end, int num_max_points,
                    int search_radius, int thr_mean, int thr_std, svs_match_result *out, int *num_new_feat_matched,
                    int *num_obs);

/* processMatchedPoints (stereo_frontend.cpp:834-974) on the results of the last svs_match or svs_match_track:
 * entry i (matched) passes when, with uvu_pred = SE3XYZ_STEREO::map(T_cur_from_actkey, xyz_actkey) on `cam`
 * (level 0), |du|, |dv| < max_reproj_error * 2^anchor_level (a float product) and |du_right| < 3. * max_reproj_error;
 * `abs` is read as the floating-point overload, as in svs_globalLoopClosure.  n_new is the candidate-index boundary
 * between new points and tracks (num_new_feat_matched's group_end).  Writes the gated entries in match order to out
 * (room for the n candidates of the last match; may be NULL), the statistics, the 3x3 add flags of addNewKeyframe
 * (add_flags[3 * i + j] = grid3x3[i][j] <= min_num_points; may be NULL) and *drop_keyframe =
 * svs_shallWeDropNewKeyframe(stats, T_cur_from_actkey, params) (may be NULL).  The gated points stay on the device as
 * the per-level point tree at uv_pyr = uvu.xy / 2^anchor_level, with the flags and num_matched_points, for
 * svs_addMorePoints(fresh = 0) until the next match.  Returns the number of gated entries, SVS_ERR_STATE when the last
 * match was not svs_match / svs_match_track on this handle, or another negative SVS_ERR_*; a refused call changes
 * nothing. */
int svs_processMatchedPoints(svs_matcher *h, const double T_cur_from_actkey[7], const svs_cam *cam, int n_new,
                             const svs_frontend_params *params, svs_tracked_point *out, svs_point_stats *stats,
                             int add_flags[9], int *drop_keyframe);

/* shallWeDropNewKeyframe (stereo_frontend.cpp:512-528): more than featureless_corners_thr quadrants with fewer than 15
 * points, or |t(T_cur_from_actkey)| > parallax_thr, or av_track_length > 75.  Plain host code.  Returns 1 (drop) or 0,
 * and SVS_ERR_INVALID (negative, so not usable as a boolean) when an argument is NULL. */
int svs_shallWeDropNewKeyframe(const svs_point_stats *stats, const double T_cur_from_actkey[7],
                               const svs_frontend_params *params);

/* addMorePointsToOtherFrame (stereo_frontend.cpp:724-823) on the current frame of the matcher, for each level l:
 *   a corner (u, v) of the level's FAST corners is taken when disp = disp0[v<<l][u<<l] * 2^-l > 0, (u<<l, v<<l) is in
 *   the level-0 frame with border 1, the add flag of its 3x3 cell (thirds as in svs_point_stats, on u<<l, v<<l) is set
 *   and the window Rect_<double>(u-R, v-R, 2R+1, 2R+1) holds no point of the level's tree (so a point at x-R is inside,
 *   one at x+R+1 is not).  A taken corner joins the tree.  Level l keeps its taken corners until one makes
 *   num_points_in[l] + kept exceed cap = num_max_points >> l (pyrFromZero_i of VisionTools, which is not vendored, is
 *   assumed to be that shift), so it keeps min(taken, max(1, cap + 1 - num_points_in[l])).
 *   fresh = 1: addNewPoints (the first frame): empty trees, every flag set, num_points_in = 0.  fresh = 0:
 *   addMorePoints: the trees, flags and num_matched_points of the last svs_processMatchedPoints, which the call reads
 *   and does not change; SVS_ERR_STATE when there was none since the last match.
 * Order (a DEVIATION): the reference walks QuadTree::EquiIter (quadtree.h:163-336), which draws from Sample::uniform.
 * The stand-in keeps its structure with a seeded hash.  With sm(x) = SplitMix64 (x += 0x9E3779B97F4A7C15;
 * z = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9; z = (z ^ (z >> 27)) * 0x94D049BB133111EB; return z ^ (z >> 31)) and
 * H(a, b, c, d, e) = sm(sm(sm(sm(sm(a) ^ b) ^ c) ^ d) ^ e) on uint64:
 *   the tree is the regular midpoint quadtree over [0, w_l) x [0, h_l) (children split at x + width * 0.5 in double;
 *   the reference's adaptive tree has the same non-empty nodes); a node's path holds two bits per depth from the root,
 *   (u >= x_mid) << 1 | (v >= y_mid), the first step highest.  Of corners at one position only the first (lowest
 *   index) exists, as in the reference's tree (delta 1).  At depth d = 0, 1, ... every node that holds a corner not
 *   yet emitted emits the one with the smallest key H(seed, 0, l, u, v) (ties: lower corner index); the nodes of one
 *   depth emit in the order of H(seed, 1, l, d, path), ties by path.  The corners are processed in emission order.
 * Outputs are in seeding order, level by level: points (may be NULL), the same as svs_match_point rows with
 * keyframe = keyframe_slot, anchor_level = l, xyz_anchor = xyz, anchor_obs_pyr = uv_pyr (may be NULL), and counts[l]
 * (SVS_MATCH_MAX_LEVELS entries, may be NULL).  The reference's push_front keeps them in reverse in newpoint_map: a
 * caller who wants its later match order reverses each call's rows.  cap (the room of points / rows) must be at least
 * the sum over levels of (num_max_points >> l) + 1.  Levels wider or taller than 65535 are SVS_ERR_UNSUPPORTED.
 * Returns the number of points or a negative SVS_ERR_*; a refused call changes nothing. */
int svs_addMorePoints(svs_matcher *h, int fresh, const double T_newkey_from_cur[7], const svs_cam *cam, int keyframe_slot,
                      const svs_frontend_params *params, svs_new_point *points, svs_match_point *rows, int cap,
                      int *counts);


/* ------------------------------------------------------------------ frame preprocessing ("next" row, SURVEY 8f) */

typedef struct svs_prep svs_prep;
/* FrameGrabber::preprocessing (frame_grabber.cpp:287-336): uint8 pyramid (cv::buildPyramid), float
 * image / 255, float pyramid (cv::gpu::pyrDown), x/y derivatives ([-1 0 1], replicated border,
 * frame_grabber.cpp:104-115) for `nlevels` levels; everything stays on the device. */
int svs_prep_create(int device, int w, int height, int nlevels, svs_prep **out);
void svs_prep_destroy(svs_prep *h);
const char *svs_prep_last_error(const svs_prep *h);
int svs_prep_process(svs_prep *h, const unsigned char *img, int pitch);
/* device pointers of one level (any output pointer may be NULL) */
int svs_prep_level(svs_prep *h, int level, int *w, int *height, const unsigned char **u8, int *pitch_u8,
                   const float **f32, const float **dx, const float **dy, int *stride_f32);
int svs_prep_get_u8(svs_prep *h, int level, unsigned char *out);          /* tightly packed w*h */
int svs_prep_get_f32(svs_prep *h, int level, int which, float *out);      /* which: 0 image, 1 dx, 2 dy */
/* device-to-device hand-over into the consumers */
int svs_dt_set_images_device(svs_dt *h, int level, const float *prev, const float *cur, const float *dx,
                             const float *dy, int stride_floats);
int svs_dt_swap_prev_cur(svs_dt *h);
int svs_matcher_set_pyramid_device(svs_matcher *h, int which, const double T_me_from_w[7],
                                   const unsigned char *const *d_pyr, const int *pitch);

/* ------------------------------------------------------------------ stereo disparity */

typedef struct svs_stereo svs_stereo;
/* calcDisparityCpu (stereo_frontend.cpp:620-653) and method 1 of calcDisparityGpu (:539-565): cv::StereoBM with the
 * reference's settings -- preFilterCap 31 (x-Sobel pre-filter), SADWindowSize 7, minDisparity 0, textureThreshold 10,
 * uniquenessRatio 15, speckleWindowSize 100, speckleRange 32, disp12MaxDiff 1 -- and numberOfDisparities =
 * num_disparities (16 * ui.num_disp16: a multiple of 16 in 16..160, else SVS_ERR_INVALID).  The result is
 * frame_data_->disp: float, the 1/16-px fixed-point disparity / 16, -1 where a stage filtered the pixel.  It equals
 * OpenCV 4.x's StereoBM bit for bit, including its invalid border (x < num_disparities + 2, x >= w - 3, three rows top
 * and bottom).  An image at most num_disparities + 5 wide, or at most 6 rows high, has no valid pixel: the map is all
 * -1 (OpenCV returns -1 up to num_disparities - 1 columns and leaves wider such maps unwritten).
 * Deviations from the reference: it links OpenCV 2.4.2; whether 2.4's StereoBM differs from 4.x's is not verified.
 * The default of the reference's CUDA build, method 2 (cv::gpu::StereoBM_GPU: another algorithm, integer output, 0 for
 * invalid), methods 3 and 4 (BP, CSBP) and the color_disp visualisation are not provided.
 * Buffers are sized at create for w x height; w and height above 65535, or w * height of 2^31 or more, are
 * SVS_ERR_INVALID. */
int svs_stereo_create(int device, int w, int height, int num_disparities, svs_stereo **out);
void svs_stereo_destroy(svs_stereo *h);
const char *svs_stereo_last_error(const svs_stereo *h);
/* left = cur_left().pyr_uint8[0], right = right.uint8 (uint8, w x height, `pitch` bytes per row).  *_on_device != 0:
 * the image is device memory of the handle's device (e.g. svs_prep_level 0), else SVS_ERR_INVALID; so is a pitch
 * smaller than w.  A refused call keeps the previous map.  Returns when the map is complete. */
int svs_stereo_compute(svs_stereo *h, const unsigned char *left, int left_pitch, int left_on_device,
                       const unsigned char *right, int right_pitch, int right_on_device);
/* the map on the device: *d_disp with *stride_floats floats per row; valid until the next compute or destroy */
int svs_stereo_disparity(svs_stereo *h, const float **d_disp, int *stride_floats);
int svs_stereo_get(svs_stereo *h, float *out);   /* w*height, tightly packed */
/* device-to-device hand-over of a level-0 disparity map into the consumers (the host setters stay as they are).
 * The map must be device memory of the consumer's device, else SVS_ERR_INVALID and the consumer keeps its map.  Each
 * returns when the copy is done, so the source may then change. */
int svs_dt_set_disparity_device(svs_dt *h, const float *d_disp, int stride_floats, int w, int height);
int svs_dtc_set_disparity_device(svs_dtc *h, const float *d_disp, int stride_floats);
int svs_matcher_set_disparity_device(svs_matcher *h, const float *d_disp, int pitch_floats);

/* ------------------------------------------------------------------ motion-only pose refinement
 * ("next" row, SURVEY.md 8f-1).  BA_SE3_XYZ_STEREO::calcFastMotionOnly (pose_optimizer.h:135-298) with
 * SE3XYZ_STEREO (transformations.h:414-460): 6-DoF Levenberg-Marquardt over fixed 3-D points with the
 * pseudo-Huber reweighting; callers stereo_frontend.cpp:1058, backend.cpp:754-779. */

typedef struct svs_pose svs_pose;

/* PoseOptimizerParams (pose_optimizer.h:38-58); SVS_POSE_PARAMS_DEFAULT mirrors its constructor */
typedef struct {
  int robust_kernel;
  double kernel_param;
  int num_iter;
  double initial_mu;   /* -1: tau * max diag(J^T J) */
  double tau;
} svs_pose_params;
#define SVS_POSE_PARAMS_DEFAULT {1, 1.0, 50, -1.0, 0.00001}

/* OptimizerStatistics (pose_optimizer.h:60-98) + counters */
typedef struct {
  double initial_chi2, chi2, max_err;
  int num_obs;
  int iterations;   /* accepted steps */
  int trials;       /* 6x6 solves */
  float ms;         /* device time of the LM kernel */
} svs_pose_stats;

int svs_pose_create(int device, int max_obs, svs_pose **out);
void svs_pose_destroy(svs_pose *h);
const char *svs_pose_last_error(const svs_pose *h);
/* obs_list as (point_id, obs = (u, v, u_right)) arrays, point_list as xyz[3 * npoints]; T_frame in/out.
 * Returns SVS_OK or a negative SVS_ERR_* (SVS_ERR_NUMERIC where the reference throws). */
int svs_calcFastMotionOnly(svs_pose *h, int n, const int *obs_point_id, const double *obs_uvu, int npoints,
                           const double *point_xyz, const svs_cam *cam, const svs_pose_params *params,
                           double T_frame[7], svs_pose_stats *stats);
/* Same, on the TrackData of the last svs_match(m, ...) where it lies on the device (matched entries'
 * obs / xyz_actkey): no host trip between matching and pose refinement. */
int svs_calcFastMotionOnly_matched(svs_pose *h, svs_matcher *m, const svs_cam *cam, const svs_pose_params *params,
                                   double T_frame[7], svs_pose_stats *stats);
/* svs_calcFastMotionOnly for a track that already lies in GPU memory: obs_point_id, obs_uvu and point_xyz are device
 * pointers on the handle's device (cam, params and T_frame stay host memory).  They are copied device to device into
 * the handle's buffers; the point_id range is checked on the device and reported with the same code and message.  The
 * result is bit-identical to svs_calcFastMotionOnly's on the same numbers.  A host pointer or memory of another
 * device gives SVS_ERR_INVALID before anything is enqueued.  The arrays are read on the handle's stream, which does
 * not wait for other streams: the caller must have finished producing them; they may be reused once the call returns. */
int svs_calcFastMotionOnly_device(svs_pose *h, int n, const int *obs_point_id, const double *obs_uvu, int npoints,
                                  const double *point_xyz, const svs_cam *cam, const svs_pose_params *params,
                                  double T_frame[7], svs_pose_stats *stats);

/* Gradient of a loss of the refined pose with respect to the observations, the points and the camera of the last
 * calcFastMotionOnly (the adjoint of the refinement), for a caller who trains keypoints, a matcher or the map's points
 * through the tracked pose.
 *   State: the inputs, parameters and returned pose T* of the last successful svs_calcFastMotionOnly or
 *     svs_calcFastMotionOnly_device call on this handle, which must have converged.
 *   Notation: f_i = z_i - pi(T X_{p_i}) the stereo residual of observation i (z_i = obs_uvu[i], X_p = point_xyz[p],
 *     p_i = obs_point_id[i]); J_i = df_i/d delta (SE3XYZ_STEREO::frameJac) for T <- exp(delta) T, delta = (upsilon,
 *     omega); r_i = max(1e-10, |f_i|), b = kernel_param and w_i = sqrt(rho(r_i)) / r_i the reweighting of
 *     pose_optimizer.h:224-231 (w_i = 1 without robust_kernel).
 *   What is differentiated: the LM stops where its right-hand side vanishes, so T* is the root of
 *     F(T) = sum_i J_i^T w_i f_i -- not the minimiser of sum_i rho(r_i), which differs on tracks with outliers.  With
 *     W_i = d(w_i f_i)/df_i = I for r_i < b (or without robust_kernel) and w_i (I - (r_i - b)/(2 r_i - b) f^_i f^_i^T)
 *     beyond, H = sum_i J_i^T W_i J_i, and (H + lambda I) v = dL_dT:
 *       dL_dobs[i] = -W_i J_i v
 *       dL_dxyz[p] = sum_{i: p_i = p} (dpi_i/dX)^T W_i J_i v             (0 for a point nobody observes)
 *       dL_dcam    = sum_i (dpi_i/d(f, px, py, b))^T W_i J_i v
 *   Conditions:
 *   - The derivatives of J_i are dropped (Gauss-Newton, as in svs_ba_observation_grad); the reweighting's derivative
 *     W_i is kept exactly.  T_init is not differentiated: the root does not depend on the start.
 *   - lambda > 0 is needed when H is singular (n <= 2 observations).
 *   - The sums over a point's observations and over all observations run in a fixed order without atomics: repeated
 *     calls give the same bits.  The call leaves the forward state alone: a later forward call gives the same bits
 *     whether or not this one ran in between.  Its buffers are allocated on its first call.
 *   Arrays: dL_dT [6] (upsilon, omega), NULL = 0; dL_dobs [n][3], dL_dxyz [npoints][3], dL_dcam [4] (f, px, py, b), in
 *   the forward's orders; a NULL output is neither computed nor written.  on_device != 0: every array is device memory
 *   of the handle's device, ready when the call is made.  The call returns after the outputs have been written.
 *   Returns 0; 1 when H + lambda I is not positive definite (the requested outputs zeroed); SVS_ERR_STATE before any
 *   successful forward call, after a failed one and after svs_calcFastMotionOnly_matched (gradients with respect to
 *   the matcher's buffers are not provided); SVS_ERR_INVALID for lambda < 0 or not finite and, with on_device, an
 *   array that is not memory of the handle's device -- all checked before anything is enqueued. */
typedef struct {
  int num_obs, npoints;
  float ms;   /* device time of the gradient kernels (the once-per-problem sort by point is not included) */
} svs_pose_grad_stats;
int svs_pose_grad(svs_pose *h, double lambda, const double dL_dT[6], double *dL_dobs, double *dL_dxyz, double *dL_dcam,
                  int on_device, svs_pose_grad_stats *stats);

/* ------------------------------------------------------------------ pose-pose constraint weights
 * ("next" row, SURVEY.md 8f-4).  SlamGraph::computeConstraint (slam_graph.cpp:785-846) for a batch of pose
 * pairs: T_1_from_2 = T_1 T_2^-1, n = number of points in both feature tables, median distance of those
 * points in frame 1, Lambda = n diag((350 |t_12| / median)^2 I3, 100^2 I3) (row-major 6x6).
 * Inputs: T_me_from_world[P][7]; the feature_table keys of every pose as CSR (feat_ptr[P+1], feat_point,
 * strictly ascending per pose); for every point the index of its anchor pose and xyz_anchor.  Anchor frames
 * outside the double window (computeAbsolutePose in the reference) are passed like any other pose.
 * A pair without shared points gets Lambda = 0 and visibility_strength = 0 (the reference calls median() of an empty
 * multiset there: undefined).  median(): VisionTools is not vendored with the reference, so its rule for an EVEN
 * number of shared points is an assumption written down here -- the mean of the two middle depths (odd n: the middle
 * one); constraint_oracle.c and csrc/constraint.cu both implement exactly this. */
typedef struct svs_constraints svs_constraints;
int svs_constraints_create(int device, svs_constraints **out);
void svs_constraints_destroy(svs_constraints *h);
const char *svs_constraints_last_error(const svs_constraints *h);
int svs_computeConstraint_batch(svs_constraints *h, int P, const double *T_me_from_world, const int *feat_ptr,
                                const int *feat_point, int L, const int *point_anchor, const double *xyz_anchor,
                                int npairs, const int *v1, const int *v2, double *T_1_from_2, double *Lambda,
                                int *visibility_strength);

/* ------------------------------------------------------------------ device-resident map and window assembly
 * ("next" row, SURVEY.md 8f-3).  The part of SlamGraph the optimiser reads (slam_graph.hpp:65-137) kept in device
 * memory -- vertices with T_me_from_world, points with anchorframe_id / xyz_anchor, observations as CSR per point
 * (vis_set order: vertex, feature centre (u, v, u_right) at level 0, pyramid level) -- and copyDataToG2o /
 * copyPosesToG2o / addPointToG2o / addObsToG2o (slam_graph.cpp:907-1032) as kernels: for the double window
 * `window_vertex` (BA pose i = vertex window_vertex[i]) and the active points (BA point l = map point
 * active_point[l]) every observation whose frame is in the window becomes an edge, in the reference's order;
 * psi = invert_depth(xyz_anchor), Lambda = diag(s, s, 0.333^2) with s = (2^-level)^2.  Observations and weights
 * never leave the device; only the index triples return to the host for the structure analysis.
 * Pose-pose constraints are passed as for svs_ba_set_problem (indices into the window). */
typedef struct svs_map svs_map;
int svs_map_create(int device, svs_map **out);
void svs_map_destroy(svs_map *h);
const char *svs_map_last_error(const svs_map *h);
int svs_map_set(svs_map *h, int V, const double *T_me_from_world, int Np, const int *point_anchor,
                const double *xyz_anchor, const int *vis_ptr, const int *vis_pose, const double *feat_center,
                const int *feat_level);
/* restoreDataFromG2o's counterpart for the map: overwrite the poses of n vertices */
int svs_map_update_poses(svs_map *h, int n, const int *vertex, const double *T_me_from_world);
/* ... and the anchored positions of n points (restoreDataFromG2o writes Point::xyz_anchor, slam_graph.cpp:1054) */
int svs_map_update_points(svs_map *h, int n, const int *point, const double *xyz_anchor);
/* read the map back (either output may be NULL): T_me_from_world[V][7], xyz_anchor[Np][3] */
int svs_map_get(svs_map *h, double *T_me_from_world, double *xyz_anchor);
/* SlamGraph::restoreDataFromG2o (slam_graph.cpp:1037-1058) device to device: after svs_ba_optimize on the window
 * svs_ba_set_problem_from_map assembled last, the vertex poses and xyz_anchor = invert_depth(psi) of its points go
 * back into the map without touching the host.
 * Refused with SVS_ERR_STATE, the map unchanged, unless `ba` still holds the very problem this map's last successful
 * svs_ba_set_problem_from_map loaded into it: after svs_map_set or svs_map_add_keyframe, after a refused
 * svs_ba_set_problem_from_map, and after any later set-up of `ba` (svs_ba_set_problem*, another map's assembly, a
 * failed set-up), even one of the same P and L, there is no window to absorb. */
int svs_map_absorb(svs_map *h, svs_ba *ba);
/* = svs_ba_set_problem on the window assembled from the map; *num_edges receives E */
int svs_ba_set_problem_from_map(svs_ba *ba, svs_map *map, int P, const int *window_vertex, const unsigned char *fixed,
                                int L, const int *active_point, int C, const int *c_i, const int *c_j,
                                const double *c_T_ji, const double *c_Lambda, const svs_cam *cam, int *num_edges);
/* The pose graph of the map: for every vertex its neighbours in the order SlamGraph::computeInitialDoubleWin pushes them
 * (Vertex::neighbor_ids_ordered_by_strength from the strongest, slam_graph.cpp:584-590; an entry in either direction is a
 * direct edge of edge_table_), and per directed entry the marginalised constraint copyContraintsToG2o reads
 * (T_nbr_from_me as qx qy qz qw tx ty tz, Lambda 6x6 row-major; both NULL when the caller brings its own constraints).
 * To be called again after svs_map_set / svs_map_add_keyframe. */
int svs_map_set_graph(svs_map *h, const int *nbr_ptr, const int *nbr_id, const double *nbr_T, const double *nbr_Lambda);
/* SlamGraph::computeInitialDoubleWin + computeActivePointsAndExtendOuterWindow (slam_graph.cpp:556-663) and the pair
 * selection of copyContraintsToG2o (:938-981) on the device tables.  Returns the double window in ascending vertex order
 * (the order of the reference's std::map; inner[i] = 1 for INNER frames; frames added by the outer-window extension are
 * OUTER), the active points in ascending order, and -- when c_i is not NULL -- the constraints between window frames of
 * which at least one is OUTER, as (c_i, c_j, T_j_from_i, Lambda) with c_i / c_j positions in window_vertex, ordered by
 * (vertex i, vertex j).  The outputs feed svs_ba_set_problem_from_map unchanged.  SVS_ERR_INVALID if a capacity is too
 * small (*P, *L, *C then hold the required sizes). */
int svs_map_select_window(svs_map *h, int root, int inner_window_size, int double_window_size, int cap_P, int *P,
                          int *window_vertex, unsigned char *inner, int cap_L, int *L, int *active_point, int cap_C, int *C,
                          int *c_i, int *c_j, double *c_T_ji, double *c_Lambda);
/* SlamGraph::addKeyframe (slam_graph.cpp:144-186) with addNewPointsToMap / addNewObsToOldPoints (:359-421) on the device
 * tables: one new vertex with T_me_from_world = T_newkey_from_oldkey * T_oldkey_from_world (composed where the map lies,
 * so a pose absorbed from the optimiser never visits the host); n_new points, each anchored in an EXISTING frame and seen
 * by that frame (new_anchor_center at level 0, new_anchor_level) and by the new keyframe (new_center, new_level); n_track
 * existing points gain an observation by the new keyframe.  The observation lists are rebuilt by kernels (count, scan,
 * move).  This call drops the pose graph: the strength bookkeeping of computeStrength / addNewEdges stays with the
 * caller, who passes the new pose graph with svs_map_set_graph, or uses svs_map_add_keyframe_graph instead.  *vertex_index = index of the new vertex, *first_new_point = index of the first new point. */
int svs_map_add_keyframe(svs_map *h, int oldkey, const double *T_newkey_from_oldkey, int n_new, const int *new_anchor,
                         const double *new_xyz_anchor, const double *new_anchor_center, const int *new_anchor_level,
                         const double *new_center, const int *new_level, int n_track, const int *track_point,
                         const double *track_center, const int *track_level, int *vertex_index, int *first_new_point);
/* ------------------------------------------------------------------ the pose graph grown on the device
 * SlamGraph::addKeyframe's computeStrength / addNewEdges (slam_graph.cpp:144-186, 424-552), registerKeyframes' METRIC
 * edges (:189-205) and addLoopClosure's APPEARANCE edge (:208-254) on the device graph, so that no caller needs a host
 * copy of the observation lists or a full graph upload after a keyframe, a registration or a loop.
 *
 * svs_map_set_pose_graph: the lists of svs_map_set_graph plus nbr_strength[nnzN], the int key of
 *   Vertex::neighbor_ids_ordered_by_strength (Edge::strength).  Each list must be non-increasing in strength (strongest
 *   first), else SVS_ERR_INVALID.  nbr_strength, nbr_T and nbr_Lambda are required (unless the graph has no entries):
 *   edges created on the device store constraints computed there.  A graph set with svs_map_set_graph has no strengths; the growth calls refuse it (SVS_ERR_STATE),
 *   as they refuse a map without a graph.
 * svs_map_get_graph: reads the graph back: nbr_ptr[V+1], nbr_id / nbr_strength [nnzN], nbr_T [nnzN][7],
 *   nbr_Lambda [nnzN][36]; any output may be NULL.  *nnzN is always set; SVS_ERR_INVALID when an entry array is asked
 *   for and cap < nnzN.  A graph without strengths reads strength 0, without constraints the identity and Lambda = 0.
 *   SVS_ERR_STATE when the map has no graph.
 * Insertion rule (std::multimap::insert, read through rbegin): a new entry of strength s goes in front of the first
 *   entry of the list with strength <= s.  Both directed entries of an edge (v1, v2) are inserted in that order: v2
 *   into v1's list, then v1 into v2's.  setConstraint(v1, v2, T_1_from_2, Lambda, Lambda): v2's entry for v1 stores
 *   T_1_from_2 (T_nbr_from_me), v1's entry for v2 stores its inverse; both store Lambda.
 * Constraints: computeConstraint(v1, v2) as svs_computeConstraint_batch computes it, on the feature tables of the
 *   map where it lies.  DEVIATION (as for svs_computeConstraint_batch): every anchor pose comes from the map; for an
 *   anchor outside the double window the reference chains computeAbsolutePose along the graph.
 *
 * svs_map_add_keyframe_graph: the whole of SlamGraph::addKeyframe.  Arguments and refusals of svs_map_add_keyframe,
 *   plus covis_thr (>= 1) and the level-0 image width, height.  In order, on the map's stream:
 *   1 computeStrength (:468-552) on the map before the growth.  New point q adds 1 to new_anchor[q].  Tracked point t,
 *     in the order given, adds 1 to every vertex of its point's observer list, and 1 to that vertex's left (else
 *     right) count when u < (int)(width * 0.5), top (else bottom) when v < (int)(height * 0.5), (u, v) =
 *     track_center[t].  QUIRK B15 (SURVEY Appendix B) is kept: the zeroing loop runs inside the track loop.  In closed
 *     form: with n_track = 0 a vertex's strength is its new-point count; otherwise it is the number of tracks t >= t*
 *     that observe it, t* the first track after which all four of its counts are present and >= covis_thr / 2
 *     (integer division), and 0 when there is no t*.  So with any track at all, new-point counts vanish.  The table
 *     holds every vertex a new point or a track touched, in ascending vertex order; then strength_to_oldkey =
 *     max(strength, covis_thr).  oldkey not in the table: SVS_ERR_INVALID (the reference asserts).
 *   2 The growth of svs_map_add_keyframe (new vertex V, new points, new observations).
 *   3 addNewEdges(LOCAL) (:424-465): every table row with strength >= covis_thr becomes the edge (v1 = row vertex,
 *     v2 = V) with that strength, its constraint computed on the grown map.  DEVIATION (a defined order): the
 *     reference walks a tr1::unordered_map; here rows are inserted in ascending vertex id, which fixes the order of
 *     equal strengths in the new vertex's list.
 *   The graph survives with V + 1 lists.  Outputs (each may be NULL): *vertex_index, *first_new_point as for
 *   svs_map_add_keyframe; table[*n_table][2] the rows (vertex, strength) after the oldkey bump (room for V rows, V
 *   before the call); *n_edges the edges added.  A refused call leaves the map and its graph bit-identical.  A CUDA
 *   error after the growth (step 3) returns SVS_ERR_CUDA with the grown map and no pose graph, as after
 *   svs_map_add_keyframe.
 *
 * svs_map_add_edges: for k = 0..n-1 the edge (v1[k], v2[k]) with strength[k] is inserted into both lists, its
 *   constraint computeConstraint(v1, v2) computed and stored by setConstraint(v1, v2, ...).  moved_vertex (or -1)
 *   is placed at T_moved_from_w[7] while the constraints are computed, as the reference does before restoring it; its
 *   map pose is not changed.  computeConstraint measures depths in v1's frame, so the callers pass:
 *     registration (registerKeyframes): v1 = stats[i].vertex of each qualified row, v2 = root, moved = root at
 *       res.T_newroot_from_w, strength = stats[i].strength;
 *     loop (addLoopClosure): v1 = loop, v2 = query, strength = res.n_tracks, moved = loop at res.T_newloop_from_w.
 *   Refused with SVS_ERR_INVALID, the map and its graph unchanged: an index outside [0, V), v1 == v2, an edge already
 *   in the graph (insertEdge asserts) or listed twice, moved_vertex outside [-1, V) or without its pose. */
int svs_map_set_pose_graph(svs_map *h, const int *nbr_ptr, const int *nbr_id, const int *nbr_strength, const double *nbr_T,
                           const double *nbr_Lambda);
int svs_map_get_graph(svs_map *h, int cap, int *nnzN, int *nbr_ptr, int *nbr_id, int *nbr_strength, double *nbr_T,
                      double *nbr_Lambda);
int svs_map_add_keyframe_graph(svs_map *h, int oldkey, const double *T_newkey_from_oldkey, int n_new, const int *new_anchor,
                               const double *new_xyz_anchor, const double *new_anchor_center, const int *new_anchor_level,
                               const double *new_center, const int *new_level, int n_track, const int *track_point,
                               const double *track_center, const int *track_level, int covis_thr, int width, int height,
                               int *vertex_index, int *first_new_point, int *n_table, int *table, int *n_edges);
int svs_map_add_edges(svs_map *h, int n, const int *v1, const int *v2, const int *strength, int moved_vertex,
                      const double *T_moved_from_w);
/* ------------------------------------------------------------------ prepareForOptimization on the device map
 * SlamGraph::prepareForOptimization(root, loop) (slam_graph.cpp:290-310) on the device graph, so that one back-end step
 * is a chain of device calls (svs_map_add_keyframe_graph -> svs_map_prepare_for_optimization ->
 * svs_ba_set_problem_from_map -> svs_ba_optimize -> svs_map_absorb) and only counts and the window reach the host.
 *
 * State.  The map keeps the window of its last prepare (the next call's old_window, WindowTable in ascending vertex order)
 *   and one Edge::is_marginalized_ flag per directed entry of the graph; both entries of an edge carry the same value.
 *   svs_map_set_graph and svs_map_set_pose_graph mark every entry marginalised and clear the window (the reference's state
 *   at its first prepare: addNewEdges and addLoopClosure end in setConstraint).  svs_map_add_keyframe_graph and
 *   svs_map_add_edges keep both: the new vertex is outside the window, new entries are marginalised, copied entries keep
 *   their flag.  svs_map_set and svs_map_add_keyframe drop the graph and the window with it.  svs_map_select_window reads
 *   the graph and changes nothing.
 *
 * svs_map_prepare_for_optimization, in order:
 *   1 The window of svs_map_select_window(root, inner_window_size, double_window_size).
 *   2 reinitializePoses (:665-725): a FIFO walk from root over the lists (strongest first).  A popped entry is skipped
 *     when its vertex was visited or is not in the NEW window.  A vertex with a parent is re-posed, T_me =
 *     getRelativePose_1_from_2(me, parent) * T_parent with T_parent the parent's updated pose, when it is marked or was
 *     not in the old window.  A vertex is marked when it is `loop` or its parent was; the mark passes to its children.
 *     getRelativePose_1_from_2 is the stored constraint of a marginalised edge, else T_me * T_parent^-1 of the current
 *     poses.  loop == root re-poses every other window vertex reachable from root; a loop outside the window, or -1,
 *     marks nothing.
 *   3 P < 2: *do_optimization = 0; the window and the poses of step 2 stay (the next call's old window is this one) and
 *     steps 4 and 5 are skipped.
 *   4 unmargPosesEnteringInnerW (:728-759): every edge whose two ends are INNER in the new window is unmarginalised.
 *   5 margPosesLeftInnerWindow (:848-904): every edge whose two ends were INNER in the old window and are not both INNER
 *     now gets computeConstraint(v1, v2) at the poses of step 2, stored as svs_map_add_edges stores it (v2's entry for
 *     v1 holds T_1_from_2, v1's entry for v2 its inverse, both Lambda) and marked marginalised.  The reference's double
 *     loop writes each such edge twice and the second write wins, so v1 = the larger and v2 = the smaller vertex index
 *     (Lambda depends on the median depth in v1's frame).
 *   Outputs: those of svs_map_select_window with its orders and capacity rules; c_T_ji / c_Lambda are read after step 5,
 *   so they go into svs_ba_set_problem_from_map unchanged.  *do_optimization = (P >= 2).  After a successful call no
 *   window waits for svs_map_absorb (its pose writes would overwrite step 2's).  One host synchronisation, for the counts.
 *   Refusals, each leaving the map, the graph and the window state bit-identical:
 *     SVS_ERR_INVALID: root outside [0, V), loop outside [-1, V), inner_window_size >= double_window_size, a null
 *       output, or a capacity too small (*P, *L, *C then hold the sizes needed; every count is found before any change);
 *     SVS_ERR_STATE: a map without a pose graph with strengths and constraints (as the growth calls).
 *   A CUDA error once the state has started to change returns SVS_ERR_CUDA with the map left without a pose graph.
 *   The lists must be symmetric (each edge has both directed entries), as every graph the growth calls build is.
 *   DEVIATIONS:
 *     anchor poses come from the map, as for svs_map_add_edges (the reference chains computeAbsolutePose for an anchor
 *       outside the new window);
 *     the vertex index stands in for the frame id: the orientation of step 5 and the std::map orders are orders of
 *       vertex index, which agree with frame ids when vertices are numbered in creation order (svs_map_add_keyframe*);
 *     both directions of a constraint are stored (the reference stores one and inverts it on read), so a re-pose through
 *       a marginalised edge can differ from the reference in the last bits;
 *     the reference asserts when copyContraintsToG2o reads an unmarginalised pair with an OUTER end (possible only after
 *       a call that stopped at P < 2); here the stored constraint is passed.
 * svs_map_get_window_state: window_type[V] (0 outside, 1 INNER, 2 OUTER: the last prepare's window) and
 *   marginalized[nnzN] (in svs_map_get_graph's entry order); either may be NULL.  *nnzN is always set; SVS_ERR_INVALID
 *   when marginalized is asked for and cap < nnzN; SVS_ERR_STATE when the map has no graph. */
int svs_map_prepare_for_optimization(svs_map *h, int root, int loop, int inner_window_size, int double_window_size,
                                     int *do_optimization, int cap_P, int *P, int *window_vertex, unsigned char *inner,
                                     int cap_L, int *L, int *active_point, int cap_C, int *C, int *c_i, int *c_j,
                                     double *c_T_ji, double *c_Lambda);
int svs_map_get_window_state(svs_map *h, int cap, int *nnzN, unsigned char *window_type, unsigned char *marginalized);
/* the edge list of the last assembly (any output may be NULL); E must equal *num_edges */
int svs_map_last_edges(svs_map *h, int E, int *e_point, int *e_pose, int *e_anchor, double *e_obs, double *e_info);

/* ------------------------------------------------------------------ metric loop verification
 * Backend::globalLoopClosure (backend.cpp:830-1001) with matchAndAlign (:726-784) on a loop that place recognition
 * proposed, from the device map, the matcher's keyframe slots and the motion-only LM, and on success
 * SlamGraph::addLoopClosure's addNewObsToOldPoints on the loop vertex (slam_graph.cpp:220, 400-420).
 *   Inputs.  query, loop: map vertex indices; T_query_from_loop: the proposal (svs_place_result).  window_vertex[P]: the
 *     double window (svs_map_select_window).  vertex_slot[V]: the matcher slot holding each vertex's keyframe pyramid,
 *     -1 = none.  The matcher's current frame must be the loop keyframe: its pyramid, its disparity and its FAST
 *     corners (recomputeFastCorners, backend.cpp:453-469).  cam: the level-0 stereo camera of the LM and the gate.
 *   1 Candidates (:844-893).  T_loop_from_world = T_query_from_loop^-1 * T_query_from_world, composed on the device
 *     from the map.  Every point the query observes whose anchor is in the window, with anchor_level and anchor_obs_pyr
 *     = centre / 2^level taken from the anchor's own observation of it, whose projection (int)(cam_vec[level].map(
 *     T_loop_from_world T_anchor^-1 xyz_anchor)) lies in the level image (border 0), in ascending point index (the
 *     reference's unordered_map order is unspecified).  Every slot then receives its vertex's map pose, loop's slot
 *     T_loop_from_world (the reference's vertex_table); the slots keep these poses after the call.
 *   2 matchAndAlign.  svs_match at radius 10 (thr_mean 22, thr_std 10) with T_cur_from_actkey = identity and
 *     T_actkey_from_w = T_loop_from_world; fewer than covis_thr matches: stage 1.  calcFastMotionOnly on the matches
 *     with PoseOptimizerParams(true, 2, 25) -> T_align1; svs_match at radius 4 from T_align1; the LM with
 *     (true, 2, 15) -> T_newloop_from_oldloop; fewer than covis_thr matches: stage 2.  A NaN residual gives
 *     SVS_ERR_NUMERIC (the reference throws).
 *   3 Gate (:904-961).  Each match is reprojected with T_newloop_from_oldloop (the projection of the LM); it becomes
 *     a track when |du|, |dv| < 2 * 2^anchor_level and |du_right| < 6.  ASSUMPTION: `abs` in backend.cpp is read as
 *     the floating-point overload; nothing in the reference tree confirms which std::abs is selected.  A track counts
 *     right when u > w/2 (else left) and lower when v > h/2 (else upper), w and h of the matcher's level 0.  Fewer
 *     than covis_thr tracks: stage 3; a quadrant with fewer than covis_thr / 2 (integer division): stage 4.
 *   4 Commit, only when verified: T_newloop_from_w = T_newloop_from_oldloop * T_query_from_loop^-1 *
 *     T_query_from_world, and each track (point, uvu at level 0, anchor_level) becomes an observation of `loop` at
 *     its ascending-vertex position in the point's list; where loop already observes the point its observation stays
 *     (std::map::insert), the track is still listed and counted.  Like svs_map_add_keyframe this forgets the last
 *     assembled window; the pose graph stays (V is unchanged).  The neighbour lists, the edge and the loop constraint
 *     are one svs_map_add_edges call (v1 = loop, v2 = query, moved = loop at T_newloop_from_w, INTEGRATION.md).
 *   Output.  res: the counts of every stage reached; tracks: track_point / track_uvu [.][3] / track_level, in match
 *     order, whenever the gate ran (cap >= n_candidates always suffices).  Returns SVS_OK whether or not the loop
 *     was verified.  Device-side findings come back through one control word; the host reads counts, poses and
 *     the track list only.
 *   Refused with SVS_ERR_INVALID, the map and the slots as they were: a NULL argument, an index outside [0, V),
 *     query == loop, covis_thr < 1, a window vertex listed twice, a slot outside the matcher or used twice, handles
 *     on different devices, a candidate whose anchor has no slot, no observation of the point or a level the matcher
 *     lacks, more candidates than the matcher's max_points or the pose handle's max_obs, and cap < n_tracks (the
 *     sizes needed are in res).  The message is in svs_map_last_error. */
typedef struct {
  int verified;                  /* the map was updated */
  int stage;                     /* 0 verified; 1 first match < covis_thr; 2 second match < covis_thr;
                                    3 gated tracks < covis_thr; 4 a quadrant < covis_thr / 2 */
  int n_candidates, n_matched1, n_matched2, n_tracks;
  int num_left, num_right, num_upper, num_lower;
  double T_align1[7];            /* T_newloop_from_oldloop after the first LM */
  double T_newloop_from_oldloop[7], T_newloop_from_w[7];   /* defined when verified */
  svs_pose_stats lm[2];
} svs_loop_result;
int svs_globalLoopClosure(svs_map *map, svs_matcher *m, svs_pose *po, const svs_cam *cam, int covis_thr, int query,
                          int loop, const double T_query_from_loop[7], int P, const int *window_vertex,
                          const int *vertex_slot, svs_loop_result *res, int cap, int *track_point, double *track_uvu,
                          int *track_level);

/* ------------------------------------------------------------------ local re-registration of a keyframe
 * Backend::localRegisterFrame (backend.cpp:549-784): the root keyframe is matched against the frames of its
 * neighbourhood that are not yet its neighbours, from the device map, its pose graph and the matcher's keyframe slots,
 * and on success SlamGraph::registerKeyframes' addNewObsToOldPoints on the root vertex (slam_graph.cpp:189-205, 400-420).
 *   Inputs.  The pose graph must be set (svs_map_set_graph), else SVS_ERR_STATE.  root: a map vertex index.
 *     window_vertex[P]: the double window (svs_map_select_window).  vertex_slot[V]: the matcher slot holding each
 *     vertex's keyframe pyramid, -1 = none.  The matcher's current frame must be the root keyframe: its pyramid, its
 *     disparity and its FAST corners re-detected on the stored cells (recomputeFastCorners, backend.cpp:453-469).
 *     po: the pose handle; cam: the level-0 stereo camera of the LM and the gate; covis_thr: graph_.covis_thr().
 *   1 Neighbourhoods and candidates (:433-449, :472-546, slam_graph.cpp:105-140).  direct = root and every vertex of
 *     root's neighbour list.  The neighbourhood framesInNeighborhood(root, |direct| + 40) is a BFS from root over the
 *     neighbour lists in their stored order (strongest first): the queue may hold a vertex more than once, a vertex
 *     outside the window is dropped when it is popped, and the BFS stops once the set has |direct| + 40 vertices.  Root
 *     outside the window gives an empty neighbourhood.  A point is a candidate when a frame of neighbourhood \ direct
 *     observes it, its anchor is in the window, and (int)(cam_vec[anchor_level].map(T_root_from_w T_anchor^-1
 *     xyz_anchor)) lies in the level image (border 0; no depth test, as in the reference).  anchor_level and
 *     anchor_obs_pyr = centre / 2^level come from the anchor's own observation of the point.  Candidates are in
 *     ascending point index (the reference's unordered_set order is unspecified).  Fewer than covis_thr: stage 1.
 *   2 matchAndAlign (:725-784).  Every slot receives its vertex's map pose (no vertex gets a predicted pose) and keeps
 *     it after the call.  svs_match at radius 10 (thr_mean 22, thr_std 10) with T_cur_from_actkey = identity and
 *     T_actkey_from_w = root's map pose; fewer than covis_thr matches: stage 2.  calcFastMotionOnly with
 *     PoseOptimizerParams(true, 2, 25) -> T_align1; svs_match at radius 4 from T_align1; the LM with (true, 2, 15)
 *     -> T_newroot_from_oldroot; fewer than covis_thr matches: stage 3.  A NaN residual gives SVS_ERR_NUMERIC.
 *   3 keyframesToRegister (:615-722).  Each match reprojected with T_newroot_from_oldroot is kept as a track when
 *     |du|, |dv| < 2 * 2^anchor_level and |du_right| < 6 (svs_globalLoopClosure's test).  Each track counts towards
 *     every vertex that observes its point, anchors a candidate and is not in direct: strength, and with the
 *     reference's names num_left when u > w/2 (else num_right), num_lower when v > h/2 (else num_upper), w and h of the
 *     matcher's level 0.  A counted vertex qualifies when strength >= covis_thr and each of the four counts >=
 *     covis_thr / 2 (integer division).  No vertex qualifies: stage 4.
 *   4 Commit (registerKeyframes' addNewObsToOldPoints).  Every track whose point a qualifying vertex observes becomes an
 *     observation of root (uvu at level 0, anchor_level) at its ascending-vertex position, once per point; where root
 *     already observes the point its observation stays.  Root's map pose is not changed (the reference restores it);
 *     T_newroot_from_w = T_newroot_from_oldroot * T_root_from_w is returned.  Like svs_map_add_keyframe this forgets
 *     the last assembled window; the pose graph stays.  addNewEdges is one svs_map_add_edges call: v1 = each
 *     qualified stats vertex, v2 = root, moved = root at T_newroot_from_w (INTEGRATION.md).
 *   Output.  res: the counts of every stage reached.  stats[n_stats]: one row per counted vertex in ascending vertex
 *     order (the reference's ImageStatsTable order is unspecified).  tracks: track_point / track_uvu [.][3] /
 *     track_level / track_committed, in match order (the reference's trackpoint-list order is unspecified), whenever
 *     the gate ran.  cap_stats >= V and cap_tracks >= n_candidates always suffice.  Returns SVS_OK whether or not the
 *     frame was registered; a rejection (stages 1-4) leaves the map bit-identical.  The host reads counts, poses and
 *     the small outputs only.
 *   Refused with SVS_ERR_INVALID, the map and the slots as they were: a NULL argument, root outside [0, V),
 *     covis_thr < 1, a window vertex listed twice, a slot outside the matcher or used twice, handles on different
 *     devices, a candidate whose anchor has no slot, no observation of the point or a level the matcher lacks, more
 *     candidates than the matcher's max_points or the pose handle's max_obs, and cap_stats < n_stats or
 *     cap_tracks < n_tracks (the sizes needed are in res).  The message is in svs_map_last_error. */
typedef struct {
  int registered;                /* the map was updated */
  int stage;                     /* 0 registered; 1 candidates < covis_thr; 2 first match < covis_thr; 3 second match <
                                    covis_thr; 4 no vertex qualifies */
  int n_direct, n_neighborhood, n_candidates, n_matched1, n_matched2;
  int n_tracks;                  /* the gated matches */
  int n_stats;                   /* the vertices keyframesToRegister counted */
  int n_neighbors;               /* the qualifying vertices */
  int n_committed;               /* the tracks committed to root */
  double T_align1[7];            /* T_newroot_from_oldroot after the first LM */
  double T_newroot_from_oldroot[7], T_newroot_from_w[7];   /* the latter defined when registered */
  svs_pose_stats lm[2];
} svs_register_result;
typedef struct {
  int vertex, strength, num_left, num_right, num_upper, num_lower;
  int qualified;
} svs_register_stats;
int svs_localRegisterFrame(svs_map *map, svs_matcher *m, svs_pose *po, const svs_cam *cam, int covis_thr, int root, int P,
                           const int *window_vertex, const int *vertex_slot, svs_register_result *res, int cap_stats,
                           svs_register_stats *stats, int cap_tracks, int *track_point, double *track_uvu,
                           int *track_level, int *track_committed);

/* ------------------------------------------------------------------ place recognition
 * PlaceRecognizer::addLocation (placerecognizer.cpp:206-324) after the caller's SURF step: vocabulary words, TF-IDF
 * loop candidates (calcLoopStatistics, :131-172) and geometricCheck (:175-202) = BFMatcher(NORM_L2).match +
 * RanSaC<SE3Model>::compute (ransac.cpp:29-137, ransac_models.cpp:27-181), one call per keyframe with no host round
 * trip between the stages.  The handle keeps the vocabulary, the stereo camera and the database of places on its
 * device; SURF detection / description, interpolateDisparity and the monitor's queue policy stay with the caller.
 *
 *   Distance.  Both nearest-neighbour searches use d = fp32 sum over dimensions 0..63 in order of
 *     d = fmaf(q - t, q - t, d) from 0.  OpenCV sums in a vectorised order, so indices equal OpenCV's except at
 *     near-ties.
 *   Words.  Row r gets the word with the smallest d (ties to the lowest index) when that d < 0.1f, else none (-1):
 *     FLANN's L2<float> is squared and radiusSearch(.., 0.1, ..) with one result slot keeps the nearest word.
 *     DEVIATION: the search is exhaustive; the reference's k-means tree (default SearchParams) is approximate, so a
 *     row may receive a closer word than the reference found.  Whether FLANN's radius test is < or <= is unverified;
 *     this is <.  number_of_words of a place = its rows that received a word.
 *   Scores (bit-exact in float, as the reference computes them).  L = places stored before the call.  Rows r of the
 *     new keyframe in order; for word w of r, every stored place k not in the exclude set holding w gets
 *       score[k] += (float(n_w(k)) / float(nwords(k))) * (float(L) / float(c_w(r)))
 *     rounded per product and summed in r order without contraction; c_w(r) = places holding w, counting the new
 *     keyframe once an earlier row of it took w (the reference inserts into inverted_index_ per descriptor).
 *     Only with do_loop_detection; the place is inserted in every case.  best = the largest score > 2, ties to the
 *     smallest keyframe id (the reference's tie order is unordered_map iteration: unspecified).
 *   Match.  Every query row is matched to the candidate's row with the smallest d (ties to the lowest index,
 *     BFMatcher::match with crossCheck = false); dist = sqrtf(d).
 *   RANSAC.  Query observations = the new uvu; train points = the candidate's xyz = unmap_uvu(uvu), computed at
 *     insertion with the handle's camera.  Hypothesis h draws match indices from its own SplitMix64 stream (state
 *     seed ^ (0xD1B54A32D192ED03 * (h + 1)); per draw state += 0x9E3779B97F4A7C15 and the standard finaliser;
 *     index ((z >> 32) * nmatch) >> 32) with the reference's redraw rules (an index equal to an earlier one of the
 *     triple is redrawn; a repeated query or train index restarts the triple).  DEVIATION: a hypothesis is void
 *     after 64 draws (the reference loops forever with fewer than three distinct train indices).  calc_motion =
 *     Kabsch with H = sum p1 p0^T on the centred triple and the determinant fix (rank(H) <= 2: U's third column is
 *     u1 x u2; a collinear triple gives NaN and no inliers); belowThreshold on map_uvu in double, T applied as its
 *     rotation matrix.  The kept hypothesis has the most inliers, ties to the lowest h; with none, T = identity
 *     (the reference's default SE3) and the inliers are those of the identity, as in the reference's last loop.
 *     nmatch < 3: 0 inliers and the identity.  Inliers are listed in match (query row) order.  A row with
 *     u == u_right gives NaN and poisons only the hypotheses that draw it.
 *   Refused with SVS_ERR_INVALID before anything is enqueued, the database untouched: a keyframe id already stored
 *     (DEVIATION: the reference would count the repeated keyframe's words in the inverted index again and keep
 *     the first place), n < 0, a NULL array with n > 0, n_exclude < 0 or
 *     a NULL exclude_ids with n_exclude > 0, num_ransac < 0, pixel_thr <= 0 or not finite.
 *   Arrays: words [W][64], desc [n][64], uvu [n][3] = (u, v, u - disparity); inlier_query / inlier_train receive
 *   num_inliers entries (room for n; NULL = not written).  p = NULL takes SVS_PLACE_PARAMS_DEFAULT. */
typedef struct svs_place svs_place;
typedef struct {
  int num_ransac;
  double pixel_thr;
  unsigned long long seed;
} svs_place_params;
#define SVS_PLACE_PARAMS_DEFAULT {100, 2.5, 0}
typedef struct {
  int best_keyframe_id;      /* argmax of the TF-IDF score, -1 if no score > 2 (or no loop detection) */
  float best_score;
  int num_matches, num_inliers;
  int loop_found;            /* num_inliers > 30: geometricCheck would call monitor.addLoop */
  double T_query_from_loop[7];
  float ms;                  /* device time of the call */
} svs_place_result;
int svs_place_create(int device, int num_words, const float *words, const svs_cam *cam, svs_place **out);
void svs_place_destroy(svs_place *h);
const char *svs_place_last_error(const svs_place *h);
int svs_place_add_location(svs_place *h, int keyframe_id, int n, const float *desc, const double *uvu,
                           int do_loop_detection, int n_exclude, const int *exclude_ids, const svs_place_params *p,
                           svs_place_result *res, int *inlier_query, int *inlier_train);
/* number of stored places */
int svs_place_num_places(const svs_place *h);
/* Read-back of the last call's intermediates, for tests and callers who keep their own policy.  Each returns a
 * count or a negative SVS_ERR_*.  words: [n], -1 = no word.  scores: the places that received a contribution, in
 * insertion order (at most cap written; the count is returned).  matches: [num_matches] (0 without a candidate).
 * hypotheses: triple [cap][3] of match indices (-1 for a void hypothesis) and inliers [cap] (-1 = void); *best = the
 * kept hypothesis or -1; returns the number run. */
int svs_place_last_words(const svs_place *h, int *word);
int svs_place_last_scores(const svs_place *h, int cap, int *keyframe_id, float *score);
int svs_place_last_matches(const svs_place *h, int *train_idx, float *dist);
int svs_place_last_hypotheses(const svs_place *h, int cap, int *triple, int *inliers, int *best);

/* Library/device info: writes "name;sm;SMs;..." into buf. */
int svs_device_info(char *buf, int buflen);

#ifdef __cplusplus
}
#endif
#endif /* SVS_B200_H */
