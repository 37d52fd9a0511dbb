/* oracle/frontend_oracle.h -- CPU restatement of the tracked frame's bookkeeping of StereoFrontend (matchAndTrack's
 * budget, processMatchedPoints, shallWeDropNewKeyframe, addMorePointsToOtherFrame); test infrastructure only.  The
 * records have the layout of their svs_* counterparts in include/svs_b200.h. */
#ifndef SVS_FRONTEND_ORACLE_H
#define SVS_FRONTEND_ORACLE_H
#include "match_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  int num_matched_points[OMATCH_MAX_LEVELS];
  int grid2x2[2][2];
  int grid3x3[3][3];
  double av_track_length;
  int num_tracked, num_new;
} ofront_stats;

typedef struct {
  int index, is_new, anchor_level, reserved;
  double uvu[3];
} ofront_tracked;

typedef struct {
  int level, reserved;
  double uv_pyr[2];
  double uvu_pyr[3];
  double xyz[3];
  double normal[3];
} ofront_new_point;

/* the stop rule of matchAndTrack on the results of all candidates (in place) */
void ofront_budget(omatch_result *res, int n_groups, const int *group_end, int num_max_points, int *num_new,
                   int *num_obs);
/* processMatchedPoints; anchor_level[i] of candidate i; cam = (f, px, py, b) of level 0; returns the gated count */
int ofront_process(const omatch_result *res, const int *anchor_level, int n, int n_new, const double T[7],
                   const double cam[4], int w0, int h0, float max_err, int min_num_points, ofront_tracked *out,
                   ofront_stats *st, int flags[9]);
int ofront_drop(const ofront_stats *st, const double T[7], int featureless_corners_thr, float parallax_thr);
/* addMorePointsToOtherFrame over nlevels levels.  The order is a DEVIATION: the reference walks QuadTree::EquiIter
 * (quadtree.h:163-336), which draws from Sample::uniform.  The stand-in keeps its structure with a seeded hash: with
 * sm = SplitMix64 and H(a, b, c, d, e) = sm(sm(sm(sm(sm(a) ^ b) ^ c) ^ d) ^ e) on uint64, the tree is the regular
 * midpoint quadtree over [0, w_l) x [0, h_l) (children split at x + width * 0.5 in double; the reference's adaptive tree
 * has the same non-empty nodes), a node's path holds (u >= x_mid) << 1 | (v >= y_mid) per depth, first step highest.
 * Of corners at one position only the lowest index exists.  At depth d = 0, 1, ... every node holding a corner not yet
 * emitted emits the one of smallest key H(seed, 0, l, u, v) (ties: lower index); the nodes of a depth emit in the
 * order of H(seed, 1, l, d, path), ties by path.  Level l keeps corners until one makes num_in[l] + kept exceed
 * num_max_points >> l (pyrFromZero_i of VisionTools, not vendored, assumed to be that shift).
 * Over the levels: corners xy[l] (nkp[l]) of level l (w[l] x h[l]); level-0 disparity;
 * tree = the gated points of ofront_process (ntrk; none when fresh); num_in = its num_matched_points (fresh: zeros);
 * flags (fresh: all set).  Writes points / rows in seeding order and counts[l]; returns the total. */
int ofront_seed(int nlevels, const int *w, const int *h, const int *const *xy, const int *nkp, const float *disp,
                int disp_pitch, const ofront_tracked *tree, int ntrk, const int *num_in, const int flags[9], int R,
                int num_max_points, unsigned long long seed, const double T[7], const double cam[4], int slot,
                ofront_new_point *points, omatch_point *rows, int *counts);
/* the emission order of the seeding for one level (corner indices; corners at an earlier corner's position are left
 * out); returns its length */
int ofront_emission_order(int w, int h, int level, const int *xy, int n, unsigned long long seed, int *order);
unsigned long long ofront_hash5(unsigned long long a, unsigned long long b, unsigned long long c, unsigned long long d,
                                unsigned long long e);

#ifdef __cplusplus
}
#endif
#endif
