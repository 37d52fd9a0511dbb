/* graph_oracle.h -- CPU restatement of the pose-graph growth of SlamGraph: computeStrength (slam_graph.cpp:468-552)
 * with its literal loops, and the neighbour-list insertion + setConstraint of addNewEdges / registerKeyframes /
 * addLoopClosure (:189-254, 424-465).  TEST INFRASTRUCTURE ONLY.  PARITY UNPINNED (the reference has no test for
 * it); pinned by a literal Python transcription (tests/test_graph_oracle.py). */
#ifndef SVS_GRAPH_ORACLE_H
#define SVS_GRAPH_ORACLE_H
#ifdef __cplusplus
extern "C" {
#endif
/* computeStrength on the map's observer lists vis_ptr[Np+1] / vis_pose: the new points' anchors, then the tracks in
 * order, each followed by the zeroing loop over the whole table (quirk B15).  half_w / half_h = (int)(w * 0.5),
 * (int)(h * 0.5).  Out: in_table[V] (0/1) and strength[V] (the table; 0 where absent).  No oldkey bump. */
void ogr_compute_strength(int V, const int *vis_ptr, const int *vis_pose, int n_new, const int *new_anchor, int n_track,
                          const int *track_point, const double *track_center, int covis_thr, int width, int height,
                          int *in_table, int *strength);
/* n edges (v1[k], v2[k], s[k]) in order into a graph of gV lists (nbr_ptr[gV+1], entries strongest first with their
 * strengths, T_nbr_from_me [7], Lambda [36]) grown to V lists: std::multimap::insert of (s, v2) into v1's list, then
 * of (s, v1) into v2's, lists read through rbegin; computeConstraint(v1, v2) on poses [V][7] and the feature tables
 * feat_ptr[V+1] / feat_point (constraint_oracle.c); setConstraint(v1, v2, T_1_from_2, Lambda, Lambda).
 * Out: out_ptr[V+1], out_id / out_str [nnz + 2n], out_T [.][7], out_L [.][36]. */
void ogr_add_edges(int gV, int V, const int *nbr_ptr, const int *nbr_id, const int *nbr_str, const double *nbr_T,
                   const double *nbr_L, int n, const int *v1, const int *v2, const int *s, const double *poses,
                   const int *feat_ptr, const int *feat_point, int Np, const int *point_anchor, const double *xyz_anchor,
                   int *out_ptr, int *out_id, int *out_str, double *out_T, double *out_L);
#ifdef __cplusplus
}
#endif
#endif
