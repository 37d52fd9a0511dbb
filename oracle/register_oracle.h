/* oracle/register_oracle.h -- CPU restatement of Backend::localRegisterFrame (backend.cpp:433-449, 472-784) with
 * SlamGraph::framesInNeighborhood (slam_graph.cpp:105-140) and registerKeyframes' addNewObsToOldPoints on the root
 * vertex (:189-205, 400-420), on the map layout of svs_map and the pose graph of svs_map_set_graph.  TEST
 * INFRASTRUCTURE ONLY: built on match_oracle.c, pose_oracle.c and loop_oracle.c. */
#ifndef SVS_REGISTER_ORACLE_H
#define SVS_REGISTER_ORACLE_H
#include "loop_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  int registered, stage;               /* as svs_register_result; stage -1: refused (err says why), -2: NaN residual */
  int n_direct, n_neighborhood, n_candidates, n_matched1, n_matched2, n_tracks, n_stats, n_neighbors, n_committed;
  double T_align1[7], T_newroot_from_oldroot[7], T_newroot_from_w[7];
  opo_stats lm[2];
  int err;                             /* 1 anchor without its observation, 2 level outside the matcher, 3 anchor without slot */
  int nnz2;                            /* observations of the grown map (registered only) */
} oreg_result;

typedef struct { int vertex, strength, num_left, num_right, num_upper, num_lower, qualified; } oreg_stats;

/* nbr_ptr [V+1] / nbr_id: the neighbour lists, strongest first.  cur: the root keyframe (pyramid, disparity, FAST trees)
 * and cam_vec; kfs[nkf]: slot pyramids (their T is set here to the vertices' map poses); cam = (f, px, py, b).
 * Outputs (NULL = not written): direct / neighborhood [V] set flags, cand_point / cand [Np] in candidate order,
 * res1 / res2 [Np] the two match results, stats [V] in ascending vertex order, track_* [Np] the gated tracks in match
 * order, and the grown map vis_ptr2 [Np+1], vis_pose2 / center2 / level2 [nnz + Np]. */
void oreg_local_register_frame(const oloop_map *m, const int *nbr_ptr, const int *nbr_id, const omatch_frame *cur,
                               omatch_keyframe *kfs, int nkf, const double cam[4], int covis_thr, int root, int P,
                               const int *window_vertex, const int *vertex_slot, oreg_result *r, int *direct,
                               int *neighborhood, int *cand_point, omatch_point *cand, omatch_result *res1,
                               omatch_result *res2, oreg_stats *stats, int *track_point, double *track_uvu,
                               int *track_level, int *track_committed, int *vis_ptr2, int *vis_pose2, double *center2,
                               int *level2);

#ifdef __cplusplus
}
#endif
#endif
