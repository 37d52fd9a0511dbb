// internal.cuh -- cross-module hooks inside libsvsb200.so (not part of the C ABI)
#pragma once
#include <cuda_runtime.h>

#include "../../include/svs_b200.h"
#include "handle.cuh"

namespace svs {
#ifdef __CUDACC__
// the reprojection gate of processMatchedPoints and of the loop / registration checks: the match predicted with T
// (SE3XYZ_STEREO::map as k_pose_lm computes it, R = T's rotation, camera f, px, py, b) lies within thr_uv pixels in u
// and v and within thr_r in u_right.  Compile with -fmad=false: the oracles restate it without contraction.
__device__ __forceinline__ bool reproj_gate(const svs_match_result& r, const double R[9], const double T[7], double f, double px,
                                            double py, double b, double thr_uv, double thr_r) {
  const double X0 = r.xyz_actkey[0], X1 = r.xyz_actkey[1], X2 = r.xyz_actkey[2];
  const double x = R[0] * X0 + R[1] * X1 + R[2] * X2 + T[4];
  const double y = R[3] * X0 + R[4] * X1 + R[5] * X2 + T[5];
  const double z = R[6] * X0 + R[7] * X1 + R[8] * X2 + T[6];
  const double d0 = r.obs[0] - (f * (x / z) + px);
  const double d1 = r.obs[1] - (f * (y / z) + py);
  const double d2 = r.obs[2] - ((x - b) / z * f + px);
  return fabs(d0) < thr_uv && fabs(d1) < thr_uv && fabs(d2) < thr_r;
}
#endif

// the matcher's internals that frontend_points.cu works on (match.cu owns them)
struct FrontState;   // frontend_points.cu: the gated points (the point tree), flags and seeding scratch, allocated on first use
struct MatcherCore {
  int device, nlevels, max_pts, max_kp;
  svs_match_level lv[SVS_MATCH_MAX_LEVELS];
  cudaStream_t stream;
  svs_match_point* d_pts;          // the handle's candidate buffer
  svs_match_result* d_res;
  const int* d_kp_xy[SVS_MATCH_MAX_LEVELS];
  int nkp[SVS_MATCH_MAX_LEVELS];
  const float* d_disp;
  int disp_pitch;
  int last_n;
  int last_pts_own;                // the last match read its candidates from d_pts (svs_match / svs_match_track)
  unsigned long long match_serial; // counts every match on the handle
  FrontState** front;
  Handle* base;                    // the matcher's error text
};
__attribute__((visibility("hidden"))) void matcher_core(svs_matcher* m, MatcherCore* c);
// k_match on n candidates already in the handle's d_pts, enqueued on its stream (no wait); the results become the
// handle's last match (last_n = n) once the caller has synchronised
__attribute__((visibility("hidden"))) int match_enqueue_own(svs_matcher* m, const double T_cur_from_actkey[7],
                                                            const double T_actkey_from_w[7], int n, int search_radius,
                                                            int thr_mean, int thr_std);
__attribute__((visibility("hidden"))) void front_state_free(FrontState* s);
// device-resident results of the last svs_match on this handle (n = number of candidate points)
__attribute__((visibility("hidden"))) void matcher_device_results(svs_matcher* m, const svs_match_result** d_res, int* n,
                                                                   int* device);
// svs_ba_set_problem_device with the observations [E][3] and weights [E][3] in one buffer (in this order) on the BA
// handle's device in the caller's edge order; every other array is on that device too (no pointer checks); returns
// after the handle has consumed the arrays
__attribute__((visibility("hidden"))) int ba_set_problem_device_obs(
    svs_ba* h, int P, const double* T_qt, const unsigned char* fixed, int L, const double* psi, int E, const int* e_point,
    const int* e_pose, const int* e_anchor, const double* d_obs_info, int C, const int* c_i, const int* c_j, const double* c_T,
    const double* c_Lambda, const svs_cam* cam);
__attribute__((visibility("hidden"))) int ba_device(const svs_ba* h);
// the block solve of svs_chol6 (chol6.cu) on its internal BA handle: the device image of the problem (S, bp, bc, x,
// tbl, ctl), the handle's stream and how often the cached symbolic analysis has been reused so far
struct BaDev;
__attribute__((visibility("hidden"))) int ba_system_on_device(svs_ba* h, const BaDev** d, cudaStream_t* stream,
                                                              int* symbolic_hits);
// sets lambda = 0 and max_iters = 0 in the control block and enqueues the reduced-system solve on the handle's stream
// (no wait); *general = 1 when the global-memory solver was launched.  keep_diag = 1: the chain solver also leaves
// L_jj^-1 in BaDev::Linv, as the general one always does
__attribute__((visibility("hidden"))) int ba_solve_system(svs_ba* h, int* general, int keep_diag = 0);
// forgets the cached structure and symbolic analysis: the next set_problem analyses the pattern afresh
__attribute__((visibility("hidden"))) void ba_forget_symbolic(svs_ba* h);
// the accepted state where it lies on the BA handle's device: pose[2][P][7], psi[2][L][3] (internal landmark order),
// lm_user[L] (internal -> caller's landmark), *cur = index of the accepted buffers, the handle's stream
__attribute__((visibility("hidden"))) int ba_state_on_device(svs_ba* h, const double* const** pose, const double* const** psi,
                                                             const int** lm_user, const int** cur, cudaStream_t* stream, int* P, int* L);
// serial number of the problem the handle holds, 0 when it holds none.  A fresh value is drawn from one process-wide
// counter at the start of every set-up (svs_ba_set_problem, _device, _sharded, _from_map; same-structure reuse too),
// so two set-ups never share one and a caller that recorded it after its own set-up can tell whether that problem is
// still the one the handle holds
__attribute__((visibility("hidden"))) unsigned long long ba_problem_serial(const svs_ba* h);
// keypoints of the last svs_fast_detect* call on this handle, on its device: xy [n][2] in cell order, cell_off [ncells + 1]
__attribute__((visibility("hidden"))) void fast_device_results(svs_fast* f, const int** d_xy, const int** d_cell_off, int* ncells,
                                                                int* n, int* device);

// the matcher's shape and where its keyframe slots keep their poses: slot s's T_me_from_w[7] lies at
// (char*)slot_T + s * slot_stride on the device
struct MatcherView {
  int device, nlevels, max_kf, max_pts;
  svs_match_level lv[SVS_MATCH_MAX_LEVELS];
  double* slot_T;
  size_t slot_stride;
};
__attribute__((visibility("hidden"))) void matcher_view(svs_matcher* m, MatcherView* v);
// svs_match on candidate points that already lie on the matcher's device (read once the call is made); the results stay
// on the device for matcher_device_results / svs_calcFastMotionOnly_matched.  Returns after the kernel has finished.
__attribute__((visibility("hidden"))) int match_device(svs_matcher* m, const double T_cur_from_actkey[7],
                                                       const double T_actkey_from_w[7], const svs_match_point* d_pts, int n,
                                                       int search_radius, int thr_mean, int thr_std);
__attribute__((visibility("hidden"))) void pose_capacity(const svs_pose* h, int* device, int* max_obs);

// the device map's tables as they lie now (valid until the map is next changed) and its stream
struct MapView {
  int V, Np, nnz, device;
  cudaStream_t stream;
  const double* pose;       // [V][7]
  const int* anchor;        // [Np]
  const double* xyz;        // [Np][3]
  const int* vis_ptr;       // [Np+1]
  const int* vis_pose;      // [nnz]
  const double* center;     // [nnz][3]
  const int* level;         // [nnz]
  Handle* base;             // the map's error text
};
__attribute__((visibility("hidden"))) void map_view(svs_map* h, MapView* v);
// the pose graph of svs_map_set_graph on the map's device (nbr_ptr [V+1], nbr_id [nnzN], strongest first); false when
// none is set
__attribute__((visibility("hidden"))) bool map_graph(svs_map* h, const int** nbr_ptr, const int** nbr_id, int* nnzN);
// exclusive scan of n counts into ptr[n + 1] by one CTA on `stream` (graph.cu's k_scan)
__attribute__((visibility("hidden"))) void launch_scan(const int* cnt, int n, int* ptr, cudaStream_t stream);
// addNewObsToOldPoints (slam_graph.cpp:400-420) for an existing vertex: n distinct points (device arrays on the map's
// device, ready on its stream) gain an observation by `vertex` at its ascending-vertex position in their lists; a point
// the vertex already observes keeps its observation.  Forgets the last assembled window, keeps the pose graph.
__attribute__((visibility("hidden"))) int map_add_observations(svs_map* h, int vertex, int n, const int* d_point,
                                                               const double* d_center, const int* d_level);
// SlamGraph::computeConstraint (constraint.cu's k_compute_constraint) on npairs pairs of device arrays, enqueued on
// `stream`: poses [.][7] and feat_ptr / feat_point (each frame's points, ascending) indexed by frame, point_anchor /
// xyz indexed by point; outputs T_1_from_2 [npairs][7], Lambda [npairs][36], strength [npairs].  scratch holds
// npairs rows of scratch_stride = constraint_scratch_stride(largest feature table) doubles (none when that is 0).
__attribute__((visibility("hidden"))) int constraint_scratch_stride(int max_feat);
__attribute__((visibility("hidden"))) void launch_compute_constraint(const double* poses, const int* feat_ptr, const int* feat_point,
                                                                     const int* point_anchor, const double* xyz, int npairs,
                                                                     const int* v1, const int* v2, double* T_1_from_2,
                                                                     double* Lambda, int* strength, double* scratch,
                                                                     int scratch_stride, cudaStream_t stream);
}  // namespace svs
