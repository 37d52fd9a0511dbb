/* prepare_oracle.h -- CPU restatement of the state change of SlamGraph::prepareForOptimization (slam_graph.cpp:290-310).
 * TEST INFRASTRUCTURE ONLY.  PARITY UNPINNED (the reference has no test for it); pinned by a literal long-double Python
 * transcription (tests/prepare_reference.py, tests/test_prepare_oracle.py). */
#ifndef SVS_PREPARE_ORACLE_H
#define SVS_PREPARE_ORACLE_H
#ifdef __cplusplus
extern "C" {
#endif
/* prepareForOptimization (slam_graph.cpp:290-310) after the window is chosen: reinitializePoses (:665-725),
 * unmargPosesEnteringInnerW (:728-759) and margPosesLeftInnerWindow (:848-904) as the reference writes them, on an
 * EdgeTable of undirected edges (min id, max id) holding T_1_from_2 in min-id orientation, Lambda_1_from_2,
 * Lambda_2_from_1 and is_marginalized_, built from the directed graph nbr_ptr[V+1] / nbr_id / nbr_T (T_nbr_from_me) /
 * nbr_L / nbr_mrg (symmetric lists, strongest first).  old_type[V] / new_type[V]: the previous and the new double
 * window (0 / 1 INNER / 2 OUTER).  poses [V][7] are updated in place; the constraints use constraint_oracle.c on
 * feat_ptr[V+1] / feat_point and every anchor pose from `poses`.  When fewer than 2 vertices are in the new window
 * only reinitializePoses runs.  Out, per directed entry: out_T / out_L (an input row when its edge was not rewritten,
 * else the EdgeTable read through getConstraint_id1_from_id2(nbr, me)), out_mrg, rewritten (0 / 1). */
void opr_prepare_for_optimization(int V, const int *nbr_ptr, const int *nbr_id, const double *nbr_T, const double *nbr_L,
                                  const unsigned char *nbr_mrg, const int *old_type, const int *new_type, int root, int loop,
                                  double *poses, const int *feat_ptr, const int *feat_point, int Np, const int *point_anchor,
                                  const double *xyz_anchor, double *out_T, double *out_L, unsigned char *out_mrg,
                                  unsigned char *rewritten);
#ifdef __cplusplus
}
#endif
#endif
