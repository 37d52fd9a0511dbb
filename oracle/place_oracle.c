/* place_oracle.c -- see place_oracle.h.  TEST INFRASTRUCTURE ONLY.
 * Single-precision sums are restated operation by operation: no FMA contraction in this file (the pragma keeps it so
 * whatever CFLAGS the Makefile passes); the one fused operation, the descriptor distance, is an explicit fmaf. */
#pragma GCC optimize("fp-contract=off")
#include "place_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#define OPL_DIM 64
#define OPL_MAX_DRAWS 64
#define OPL_JACOBI_SWEEPS 32

typedef struct { int place, count; } opl_entry;
typedef struct { opl_entry *e; int len, cap; } opl_list;

struct opl_db {
  int W;
  float *words;          /* [W][64] */
  double cam[4];         /* f px py b */
  opl_list *inverted;    /* [W]: (place, count) in insertion order (inverted_index_) */
  int L, cap;
  int *id, *nwords, *nrows;
  float **desc;          /* [L] -> [nrows][64] */
  double **xyz;          /* [L] -> [nrows][3]  (unmap_uvu at insertion) */
};

/* d = sum over k = 0..63 in order of (q - t)^2, one fmaf per term */
float opl_sqdist(const float *a, const float *b) {
  float d = 0.f;
  for (int k = 0; k < OPL_DIM; ++k) {
    const float df = a[k] - b[k];
    d = fmaf(df, df, d);
  }
  return d;
}

/* nearest train row by opl_sqdist, ties to the lowest index (d[] receives the squared distance) */
void opl_nn(int n, const float *query, int m, const float *train, int *idx, float *d) {
  for (int r = 0; r < n; ++r) {
    int best = -1;
    float bd = 0.f;
    for (int j = 0; j < m; ++j) {
      const float v = opl_sqdist(query + (size_t)r * OPL_DIM, train + (size_t)j * OPL_DIM);
      if (best < 0 || v < bd) { best = j; bd = v; }
    }
    idx[r] = best;
    d[r] = bd;
  }
}

/* StereoCamera::unmap_uvu (stereo_camera.cpp:46-52) */
static void unmap_uvu(const double c[4], const double uvu[3], double xyz[3]) {
  const double sd = (uvu[0] - uvu[2]) / c[3];
  const double z = c[0] / sd;
  xyz[0] = ((uvu[0] - c[1]) / c[0]) * z;
  xyz[1] = ((uvu[1] - c[2]) / c[0]) * z;
  xyz[2] = z;
}

/* AbsoluteOrientation::belowThreshold (ransac_models.cpp:27-42) of T * X, T applied as (R, t) */
static int below_threshold(const double c[4], const double R[9], const double t[3], const double X[3],
                           const double obs[3], double thr2) {
  double p[3];
  for (int i = 0; i < 3; ++i) p[i] = ((R[3 * i] * X[0] + R[3 * i + 1] * X[1]) + R[3 * i + 2] * X[2]) + t[i];
  const double u = c[0] * (p[0] / p[2]) + c[1];
  const double v = c[0] * (p[1] / p[2]) + c[2];
  const double ur = (p[0] - c[3]) / p[2] * c[0] + c[1];
  const double du = obs[0] - u, dv = obs[1] - v, dr = obs[2] - ur;
  return du * du < thr2 && dv * dv < thr2 && dr * dr < thr2;
}

/* getOrientationAndCentriods + SE3Model::calc_motion (ransac_models.cpp:44-81, 138-169): p0 = the three query points
 * (row-major [3][3]), p1 = the three train points.  H = sum p1 p0^T on the centred triple, SVD by one-sided Jacobi;
 * a centred triple has rank(H) <= 2, so U's third column is taken as u1 x u2 and R = V U^T is unique after the
 * determinant fix (flip V's third column). */
void opl_kabsch(const double p0_in[9], const double p1_in[9], double R[9], double t[3]) {
  double p0[9], p1[9], c0[3], c1[3];
  for (int i = 0; i < 3; ++i) {
    c0[i] = ((p0_in[i] + p0_in[3 + i]) + p0_in[6 + i]) * (1.0 / 3.0);
    c1[i] = ((p1_in[i] + p1_in[3 + i]) + p1_in[6 + i]) * (1.0 / 3.0);
  }
  for (int a = 0; a < 3; ++a)
    for (int i = 0; i < 3; ++i) { p0[3 * a + i] = p0_in[3 * a + i] - c0[i]; p1[3 * a + i] = p1_in[3 * a + i] - c1[i]; }
  double A[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) A[3 * i + j] = (p1[i] * p0[j] + p1[3 + i] * p0[3 + j]) + p1[6 + i] * p0[6 + j];
  static const int P[3] = {0, 0, 1}, Q[3] = {1, 2, 2};
  for (int sweep = 0; sweep < OPL_JACOBI_SWEEPS; ++sweep) {
    int rotated = 0;
    for (int pq = 0; pq < 3; ++pq) {
      const int p = P[pq], q = Q[pq];
      const double al = (A[p] * A[p] + A[3 + p] * A[3 + p]) + A[6 + p] * A[6 + p];
      const double be = (A[q] * A[q] + A[3 + q] * A[3 + q]) + A[6 + q] * A[6 + q];
      const double ga = (A[p] * A[q] + A[3 + p] * A[3 + q]) + A[6 + p] * A[6 + q];
      if (!(fabs(ga) > 1e-15 * sqrt(al * be))) continue;   /* converged pair (or NaN: no rotation) */
      const double ze = (be - al) / (2.0 * ga);
      const double tt = (ze >= 0.0 ? 1.0 : -1.0) / (fabs(ze) + sqrt(1.0 + ze * ze));
      const double cs = 1.0 / sqrt(1.0 + tt * tt), sn = cs * tt;
      for (int i = 0; i < 3; ++i) {
        const double ap = A[3 * i + p], aq = A[3 * i + q];
        A[3 * i + p] = cs * ap - sn * aq;
        A[3 * i + q] = sn * ap + cs * aq;
        const double vp = V[3 * i + p], vq = V[3 * i + q];
        V[3 * i + p] = cs * vp - sn * vq;
        V[3 * i + q] = sn * vp + cs * vq;
      }
      rotated = 1;
    }
    if (!rotated) break;
  }
  double sg[3];
  for (int j = 0; j < 3; ++j) sg[j] = sqrt((A[j] * A[j] + A[3 + j] * A[3 + j]) + A[6 + j] * A[6 + j]);
  int o[3] = {0, 1, 2};
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2 - a; ++b)
      if (sg[o[b + 1]] > sg[o[b]]) { const int tmp = o[b]; o[b] = o[b + 1]; o[b + 1] = tmp; }
  double u1[3], u2[3], u3[3], v1[3], v2[3], v3[3];
  for (int i = 0; i < 3; ++i) {
    u1[i] = A[3 * i + o[0]] / sg[o[0]];
    u2[i] = A[3 * i + o[1]] / sg[o[1]];
    v1[i] = V[3 * i + o[0]]; v2[i] = V[3 * i + o[1]]; v3[i] = V[3 * i + o[2]];
  }
  u3[0] = u1[1] * u2[2] - u1[2] * u2[1];
  u3[1] = u1[2] * u2[0] - u1[0] * u2[2];
  u3[2] = u1[0] * u2[1] - u1[1] * u2[0];
  for (int pass = 0; pass < 2; ++pass) {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) R[3 * i + j] = (v1[i] * u1[j] + v2[i] * u2[j]) + v3[i] * u3[j];
    const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) +
                       R[2] * (R[3] * R[7] - R[4] * R[6]);
    if (!(det < 0.0)) break;
    for (int i = 0; i < 3; ++i) v3[i] = -v3[i];
  }
  for (int i = 0; i < 3; ++i) t[i] = c0[i] - ((R[3 * i] * c1[0] + R[3 * i + 1] * c1[1]) + R[3 * i + 2] * c1[2]);
}

/* Eigen's Quaternion-from-rotation-matrix (the SE3's stored rotation) */
static void quat_from_R(const double R[9], double q[4]) {
  const double tr = (R[0] + R[4]) + R[8];
  if (tr > 0.0) {
    double s = sqrt(tr + 1.0);
    q[3] = 0.5 * s;
    s = 0.5 / s;
    q[0] = (R[7] - R[5]) * s;
    q[1] = (R[2] - R[6]) * s;
    q[2] = (R[3] - R[1]) * s;
  } else {
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[3 * i + i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double s = sqrt(R[3 * i + i] - R[3 * j + j] - R[3 * k + k] + 1.0);
    q[i] = 0.5 * s;
    s = 0.5 / s;
    q[3] = (R[3 * k + j] - R[3 * j + k]) * s;
    q[j] = (R[3 * j + i] + R[3 * i + j]) * s;
    q[k] = (R[3 * k + i] + R[3 * i + k]) * s;
  }
}

unsigned long long opl_splitmix_next(unsigned long long *state) {
  unsigned long long z = (*state += 0x9E3779B97F4A7C15ULL);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}

/* The sampling loop of RanSaC::compute (ransac.cpp:68-96) with hypothesis h's own SplitMix64 stream; the match of
 * index i is (query row i, train_idx[i]).  Returns the number of draws, or -1 when the hypothesis is void (64 draws
 * without a valid triple; the reference would loop forever when fewer than three distinct train indices exist). */
int opl_draw_triple(unsigned long long seed, int h, int nmatch, const int *train_idx, int triple[3]) {
  unsigned long long st = seed ^ (0xD1B54A32D192ED03ULL * (unsigned long long)(h + 1));
  int draws = 0;
restart:
  for (int i = 0; i < 3; ++i) {
  redraw:
    if (draws == OPL_MAX_DRAWS) return -1;
    triple[i] = (int)(((opl_splitmix_next(&st) >> 32) * (unsigned long long)nmatch) >> 32);
    ++draws;
    for (int j = 0; j < i; ++j)
      if (triple[j] == triple[i]) goto redraw;
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < i; ++j)
      if (triple[i] == triple[j] || train_idx[triple[i]] == train_idx[triple[j]]) goto restart;
  return draws;
}

opl_db *opl_create(int num_words, const float *words, const double cam[4]) {
  if (num_words <= 0 || !words || !cam) return NULL;
  opl_db *db = calloc(1, sizeof *db);
  db->W = num_words;
  db->words = malloc(sizeof(float) * OPL_DIM * (size_t)num_words);
  memcpy(db->words, words, sizeof(float) * OPL_DIM * (size_t)num_words);
  memcpy(db->cam, cam, sizeof db->cam);
  db->inverted = calloc((size_t)num_words, sizeof(opl_list));
  return db;
}

void opl_destroy(opl_db *db) {
  if (!db) return;
  for (int w = 0; w < db->W; ++w) free(db->inverted[w].e);
  for (int k = 0; k < db->L; ++k) { free(db->desc[k]); free(db->xyz[k]); }
  free(db->inverted); free(db->words); free(db->id); free(db->nwords); free(db->nrows); free(db->desc); free(db->xyz);
  free(db);
}

int opl_num_places(const opl_db *db) { return db ? db->L : 0; }

static int place_of(const opl_db *db, int id) {
  for (int k = 0; k < db->L; ++k)
    if (db->id[k] == id) return k;
  return -1;
}

int opl_add_location(opl_db *db, int keyframe_id, int n, const float *desc, const double *uvu, int do_loop_detection,
                     int n_exclude, const int *exclude_ids, int num_ransac, double pixel_thr, unsigned long long seed,
                     opl_result *res, int *word_out, int *score_id, float *score_val, int *nscores, int *train_out,
                     float *dist_out, int *hyp_triple, int *hyp_inliers, int *inlier_query, int *inlier_train) {
  if (!db || !res || n < 0 || (n > 0 && (!desc || !uvu)) || n_exclude < 0 || (n_exclude > 0 && !exclude_ids) ||
      num_ransac < 0 || !(pixel_thr > 0.0) || !isfinite(pixel_thr) || place_of(db, keyframe_id) >= 0)
    return -1;
  const int L = db->L, cur = L;
  memset(res, 0, sizeof *res);
  res->best_keyframe_id = -1;
  res->best_hypothesis = -1;
  res->T_query_from_loop[3] = 1.0;
  int *word = malloc(sizeof(int) * (size_t)(n + 1));
  float *wd = malloc(sizeof(float) * (size_t)(n + 1));
  /* flann radiusSearch(query, 0.1) with one result slot: the nearest word when its distance is below the radius */
  opl_nn(n, desc, db->W, db->words, word, wd);
  for (int r = 0; r < n; ++r)
    if (!(wd[r] < 0.1f)) word[r] = -1;
  float *score = calloc((size_t)L + 1, sizeof(float));
  unsigned char *touched = calloc((size_t)L + 1, 1), *excluded = calloc((size_t)L + 1, 1);
  for (int e = 0; e < n_exclude; ++e) {
    const int k = place_of(db, exclude_ids[e]);
    if (k >= 0) excluded[k] = 1;
  }
  int nw = 0;
  for (int r = 0; r < n; ++r) {
    const int w = word[r];
    if (w < 0) continue;
    ++nw;
    opl_list *inv = &db->inverted[w];
    if (do_loop_detection && inv->len > 0) {   /* calcLoopStatistics */
      const float idf = (float)L / (float)inv->len;
      for (int e = 0; e < inv->len; ++e) {
        const int k = inv->e[e].place;
        if (k == cur || excluded[k]) continue;
        const float tf = (float)inv->e[e].count / (float)db->nwords[k];
        const float val = tf * idf;
        score[k] = score[k] + val;
        touched[k] = 1;
      }
    }
    if (inv->len > 0 && inv->e[inv->len - 1].place == cur) {
      ++inv->e[inv->len - 1].count;
    } else {
      if (inv->len == inv->cap) {
        inv->cap = inv->cap ? 2 * inv->cap : 4;
        inv->e = realloc(inv->e, sizeof(opl_entry) * (size_t)inv->cap);
      }
      inv->e[inv->len].place = cur;
      inv->e[inv->len].count = 1;
      ++inv->len;
    }
  }
  /* location_map_.insert */
  if (L == db->cap) {
    db->cap = db->cap ? 2 * db->cap : 16;
    db->id = realloc(db->id, sizeof(int) * (size_t)db->cap);
    db->nwords = realloc(db->nwords, sizeof(int) * (size_t)db->cap);
    db->nrows = realloc(db->nrows, sizeof(int) * (size_t)db->cap);
    db->desc = realloc(db->desc, sizeof(float *) * (size_t)db->cap);
    db->xyz = realloc(db->xyz, sizeof(double *) * (size_t)db->cap);
  }
  db->id[cur] = keyframe_id;
  db->nwords[cur] = nw;
  db->nrows[cur] = n;
  db->desc[cur] = malloc(sizeof(float) * OPL_DIM * (size_t)(n + 1));
  if (n) memcpy(db->desc[cur], desc, sizeof(float) * OPL_DIM * (size_t)n);
  db->xyz[cur] = malloc(sizeof(double) * 3 * (size_t)(n + 1));
  for (int r = 0; r < n; ++r) unmap_uvu(db->cam, uvu + 3 * (size_t)r, db->xyz[cur] + 3 * (size_t)r);
  db->L = L + 1;
  res->number_of_words = nw;
  if (word_out && n) memcpy(word_out, word, sizeof(int) * (size_t)n);
  int ns = 0, best = -1;
  for (int k = 0; k < L; ++k) {
    if (!touched[k]) continue;
    if (score_id) score_id[ns] = db->id[k];
    if (score_val) score_val[ns] = score[k];
    ++ns;
    /* the largest score > 2, ties to the smallest keyframe id */
    if (score[k] > 2.f && (best < 0 || score[k] > score[best] || (score[k] == score[best] && db->id[k] < db->id[best])))
      best = k;
  }
  if (nscores) *nscores = ns;
  if (best >= 0) {
    res->best_keyframe_id = db->id[best];
    res->best_score = score[best];
    /* geometricCheck: BFMatcher(NORM_L2).match, then RanSaC<SE3Model>::compute */
    const int m = db->nrows[best];
    int *tidx = malloc(sizeof(int) * (size_t)(n + 1));
    float *td = malloc(sizeof(float) * (size_t)(n + 1));
    opl_nn(n, desc, m, db->desc[best], tidx, td);
    const int nmatch = m > 0 ? n : 0;
    for (int r = 0; r < nmatch; ++r) td[r] = sqrtf(td[r]);
    res->num_matches = nmatch;
    if (train_out && nmatch) memcpy(train_out, tidx, sizeof(int) * (size_t)nmatch);
    if (dist_out && nmatch) memcpy(dist_out, td, sizeof(float) * (size_t)nmatch);
    const double thr2 = pixel_thr * pixel_thr;
    const double *xyz = db->xyz[best];
    double Rb[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, tb[3] = {0, 0, 0};
    if (nmatch >= 3) {
      int bestinl = 0;
      res->num_hypotheses = num_ransac;
      for (int h = 0; h < num_ransac; ++h) {
        int tri[3];
        const int draws = opl_draw_triple(seed, h, nmatch, tidx, tri);
        if (hyp_triple) for (int a = 0; a < 3; ++a) hyp_triple[3 * h + a] = draws < 0 ? -1 : tri[a];
        if (draws < 0) {
          if (hyp_inliers) hyp_inliers[h] = -1;
          continue;
        }
        double p0[9], p1[9], R[9], t[3];
        for (int a = 0; a < 3; ++a) {
          unmap_uvu(db->cam, uvu + 3 * (size_t)tri[a], p0 + 3 * a);
          for (int i = 0; i < 3; ++i) p1[3 * a + i] = xyz[3 * (size_t)tidx[tri[a]] + i];
        }
        opl_kabsch(p0, p1, R, t);
        int inl = 0;
        for (int r = 0; r < nmatch; ++r)
          inl += below_threshold(db->cam, R, t, xyz + 3 * (size_t)tidx[r], uvu + 3 * (size_t)r, thr2);
        if (hyp_inliers) hyp_inliers[h] = inl;
        if (inl > bestinl) {
          bestinl = inl;
          res->best_hypothesis = h;
          memcpy(Rb, R, sizeof Rb);
          memcpy(tb, t, sizeof tb);
        }
      }
      /* the inliers of the kept transformation (the identity when no hypothesis had one), in match order */
      int ni = 0;
      for (int r = 0; r < nmatch; ++r)
        if (below_threshold(db->cam, Rb, tb, xyz + 3 * (size_t)tidx[r], uvu + 3 * (size_t)r, thr2)) {
          if (inlier_query) inlier_query[ni] = r;
          if (inlier_train) inlier_train[ni] = tidx[r];
          ++ni;
        }
      res->num_inliers = ni;
    }
    quat_from_R(Rb, res->T_query_from_loop);
    for (int i = 0; i < 3; ++i) res->T_query_from_loop[4 + i] = tb[i];
    res->loop_found = res->num_inliers > 30;
    free(tidx); free(td);
  }
  free(word); free(wd); free(score); free(touched); free(excluded);
  return 0;
}
