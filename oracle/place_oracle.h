/* place_oracle.h -- CPU restatement of PlaceRecognizer::addLocation (placerecognizer.cpp:206-324) with
 * calcLoopStatistics (:131-172), geometricCheck (:175-202), RanSaC<SE3Model>::compute (ransac.cpp:29-137) and
 * SE3Model::calc_motion / belowThreshold (ransac_models.cpp:27-181), under the semantics written down in
 * include/svs_b200.h (svs_place): exhaustive words, a fixed fp32 summation order, SplitMix64 sampling per hypothesis.
 * TEST INFRASTRUCTURE ONLY.  The database is kept the way the reference keeps it: an inverted index per word of
 * (place, count) pairs filled descriptor by descriptor, and plain per-place arrays. */
#ifndef PLACE_ORACLE_H
#define PLACE_ORACLE_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct opl_db opl_db;

typedef struct {
  int best_keyframe_id;   /* -1: no score > 2 or no loop detection */
  float best_score;
  int num_matches, num_inliers, loop_found;
  double T_query_from_loop[7];   /* qx qy qz qw tx ty tz */
  int number_of_words;           /* descriptors of the new place that received a word */
  int best_hypothesis;           /* -1: none with an inlier */
  int num_hypotheses;            /* hypotheses run (0 without a candidate or with fewer than 3 matches) */
} opl_result;

opl_db *opl_create(int num_words, const float *words, const double cam[4]);
void opl_destroy(opl_db *db);
int opl_num_places(const opl_db *db);

/* Returns 0, or -1 for a refused input (the database is then untouched).  Every output may be NULL:
 * word[n]; score_id / score_val in place order for the places that received a contribution (count in *nscores);
 * train_idx[n], dist[n] of the match against the candidate; hyp_triple[3 * num_ransac] (match indices) and
 * hyp_inliers[num_ransac] (-1 = void after 64 draws); inlier_query / inlier_train [num_inliers]. */
int opl_add_location(opl_db *db, int keyframe_id, int n, const float *desc, const double *uvu, int do_loop_detection,
                     int n_exclude, const int *exclude_ids, int num_ransac, double pixel_thr, unsigned long long seed,
                     opl_result *res, int *word, int *score_id, float *score_val, int *nscores, int *train_idx,
                     float *dist, int *hyp_triple, int *hyp_inliers, int *inlier_query, int *inlier_train);

/* the building blocks, for tests */
float opl_sqdist(const float *a, const float *b);
void opl_nn(int n, const float *query, int m, const float *train, int *idx, float *d);
void opl_kabsch(const double p0[9], const double p1[9], double R[9], double t[3]);
unsigned long long opl_splitmix_next(unsigned long long *state);
int opl_draw_triple(unsigned long long seed, int h, int nmatch, const int *train_idx, int triple[3]);

#ifdef __cplusplus
}
#endif
#endif
