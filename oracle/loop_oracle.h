/* oracle/loop_oracle.h -- CPU restatement of Backend::globalLoopClosure (backend.cpp:830-1001) with matchAndAlign
 * (:726-784) and addLoopClosure's addNewObsToOldPoints on the loop vertex (slam_graph.cpp:220, 400-420), on the map
 * layout of svs_map.  TEST INFRASTRUCTURE ONLY: built on match_oracle.c and pose_oracle.c. */
#ifndef SVS_LOOP_ORACLE_H
#define SVS_LOOP_ORACLE_H
#include "match_oracle.h"
#include "pose_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct {                       /* svs_map's tables */
  int V, Np;
  const double *pose;                  /* [V][7] */
  const int *anchor;                   /* [Np] */
  const double *xyz;                   /* [Np][3] */
  const int *vis_ptr, *vis_pose;       /* [Np+1], [nnz] */
  const double *center;                /* [nnz][3] */
  const int *level;                    /* [nnz] */
} oloop_map;

typedef struct {
  int verified, stage;                 /* as svs_loop_result; stage -1: refused (err says why) */
  int n_candidates, n_matched1, n_matched2, n_tracks;
  int num_left, num_right, num_upper, num_lower;
  double T_loop_from_w[7], T_align1[7], T_newloop_from_oldloop[7], T_newloop_from_w[7];
  opo_stats lm[2];
  int err;                             /* 1 anchor without its observation, 2 level outside the matcher, 3 anchor without slot */
  int nnz2;                            /* observations of the grown map (verified only) */
} oloop_result;

/* cur: the loop keyframe (pyramid, disparity, FAST trees) and cam_vec; kfs[nkf]: slot pyramids (their T is set here by
 * the refresh rule); cam = (f, px, py, b).  Outputs (NULL = not written): cand_point / cand [Np] in candidate order,
 * res1 / res2 [Np] the two match results, track_* [Np] the gated tracks, and the grown map vis_ptr2 [Np+1],
 * vis_pose2 / center2 / level2 [nnz + Np]. */
void oloop_global_loop_closure(const oloop_map *m, const omatch_frame *cur, omatch_keyframe *kfs, int nkf, const double cam[4],
                               int covis_thr, int query, int loop, const double T_query_from_loop[7], int P,
                               const int *window_vertex, const int *vertex_slot, oloop_result *r, int *cand_point,
                               omatch_point *cand, omatch_result *res1, omatch_result *res2, int *track_point,
                               double *track_uvu, int *track_level, int *vis_ptr2, int *vis_pose2, double *center2,
                               int *level2);
/* SE3XYZ_STEREO::map as the gate evaluates it (no FMA contraction) */
void oloop_map_uvu(const double cam[4], const double T[7], const double xyz[3], double uvu[3]);
void oloop_se3_mul(const double A[7], const double B[7], double AB[7]);
void oloop_se3_inv(const double A[7], double Ai[7]);
void oloop_se3_act(const double A[7], const double x[3], double y[3]);

#ifdef __cplusplus
}
#endif
#endif
