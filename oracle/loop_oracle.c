/* loop_oracle.c -- see loop_oracle.h.  TEST INFRASTRUCTURE ONLY.  Written sequentially from backend.cpp:830-1001 and
 * slam_graph.cpp:400-420; the projections are restated operation by operation without FMA contraction (the pragma
 * keeps it so under the Makefile's flags), like csrc/loop.cu compiled with -fmad=false. */
#pragma GCC optimize("fp-contract=off")
#include "loop_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

static void quat_to_R(const double q[4], double R[9]) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w;
  const double txx = tx * x, txy = ty * x, txz = tz * x;
  const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
  R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}
static void mat3_vec(const double R[9], const double x[3], double y[3]) {
  y[0] = R[0] * x[0] + R[1] * x[1] + R[2] * x[2];
  y[1] = R[3] * x[0] + R[4] * x[1] + R[5] * x[2];
  y[2] = R[6] * x[0] + R[7] * x[1] + R[8] * x[2];
}
void oloop_se3_act(const double A[7], const double x[3], double y[3]) {
  double R[9];
  quat_to_R(A, R);
  mat3_vec(R, x, y);
  y[0] += A[4]; y[1] += A[5]; y[2] += A[6];
}
/* Sophus SE3 product with the quaternion renormalised */
void oloop_se3_mul(const double A[7], const double B[7], double AB[7]) {
  double R[9], t[3], q[4];
  quat_to_R(A, R);
  mat3_vec(R, B + 4, t);
  const double ax = A[0], ay = A[1], az = A[2], aw = A[3];
  const double bx = B[0], by = B[1], bz = B[2], bw = B[3];
  q[3] = aw * bw - ax * bx - ay * by - az * bz;
  q[0] = aw * bx + ax * bw + ay * bz - az * by;
  q[1] = aw * by + ay * bw + az * bx - ax * bz;
  q[2] = aw * bz + az * bw + ax * by - ay * bx;
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  AB[0] = q[0] / n; AB[1] = q[1] / n; AB[2] = q[2] / n; AB[3] = q[3] / n;
  AB[4] = A[4] + t[0]; AB[5] = A[5] + t[1]; AB[6] = A[6] + t[2];
}
void oloop_se3_inv(const double A[7], double Ai[7]) {
  const double q[4] = {-A[0], -A[1], -A[2], A[3]};
  const double mt[3] = {-A[4], -A[5], -A[6]};
  double R[9], t[3];
  quat_to_R(q, R);
  mat3_vec(R, mt, t);
  Ai[0] = q[0]; Ai[1] = q[1]; Ai[2] = q[2]; Ai[3] = q[3];
  Ai[4] = t[0]; Ai[5] = t[1]; Ai[6] = t[2];
}

/* SE3XYZ_STEREO::map (transformations.h:445-449, stereo_camera.cpp:36-44): x = R X + t summed left to right */
void oloop_map_uvu(const double cam[4], const double T[7], const double X[3], double uvu[3]) {
  double R[9];
  quat_to_R(T, R);
  const double x = R[0] * X[0] + R[1] * X[1] + R[2] * X[2] + T[4];
  const double y = R[3] * X[0] + R[4] * X[1] + R[5] * X[2] + T[5];
  const double z = R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + T[6];
  uvu[0] = cam[0] * (x / z) + cam[1];
  uvu[1] = cam[0] * (y / z) + cam[2];
  uvu[2] = (x - cam[3]) / z * cam[0] + cam[1];
}

/* the matched entries of one match result as calcFastMotionOnly's obs_list / point_list (TrackData order) */
static int align(int n, const omatch_result *res, const double cam[4], int num_iter, double T[7], opo_stats *st) {
  int nm = 0;
  for (int i = 0; i < n; ++i) nm += res[i].matched;
  memset(st, 0, sizeof *st);
  if (nm == 0) return 0;
  int *pid = malloc(sizeof(int) * nm);
  double *obs = malloc(sizeof(double) * 3 * nm), *pts = malloc(sizeof(double) * 3 * nm);
  int k = 0;
  for (int i = 0; i < n; ++i) {
    if (!res[i].matched) continue;
    pid[k] = k;
    memcpy(obs + 3 * k, res[i].obs, sizeof(double) * 3);
    memcpy(pts + 3 * k, res[i].xyz_actkey, sizeof(double) * 3);
    ++k;
  }
  opo_calc_fast_motion_only(nm, pid, obs, pts, cam, 1, 2.0, num_iter, -1.0, 0.00001, T, st); /* PoseOptimizerParams(true, 2, it) */
  free(pid); free(obs); free(pts);
  return st->nan_error;
}

void oloop_global_loop_closure(const oloop_map *m, const omatch_frame *cur, omatch_keyframe *kfs, int nkf, const double cam[4],
                               int covis_thr, int query, int loop, const double Tql[7], int P, const int *window_vertex,
                               const int *vertex_slot, oloop_result *r, int *cand_point, omatch_point *cand,
                               omatch_result *res1, omatch_result *res2, int *track_point, double *track_uvu, int *track_level,
                               int *vis_ptr2, int *vis_pose2, double *center2, int *level2) {
  memset(r, 0, sizeof *r);
  int nlv = 0;
  while (nlv < OMATCH_MAX_LEVELS && cur->levels[nlv].w > 0) ++nlv;
  char *inwin = calloc((size_t)m->V, 1);
  for (int i = 0; i < P; ++i) inwin[window_vertex[i]] = 1;
  const int cap = m->Np > 0 ? m->Np : 1;
  int *cp = malloc(sizeof(int) * cap);
  omatch_point *pts = malloc(sizeof(omatch_point) * cap);
  omatch_result *ra = malloc(sizeof(omatch_result) * cap), *rb = malloc(sizeof(omatch_result) * cap);
  /* :844-845 */
  double Tlq[7];
  oloop_se3_inv(Tql, Tlq);
  oloop_se3_mul(Tlq, m->pose + 7 * query, r->T_loop_from_w);
  /* :853-893 over the points the query observes, ascending */
  int nc = 0;
  for (int p = 0; p < m->Np; ++p) {
    int seen = 0, ia = -1;
    const int a = m->anchor[p];
    for (int k = m->vis_ptr[p]; k < m->vis_ptr[p + 1]; ++k) {
      if (m->vis_pose[k] == query) seen = 1;
      if (m->vis_pose[k] == a && ia < 0) ia = k;
    }
    if (!seen || !inwin[a]) continue;
    if (ia < 0) { r->err = 1; continue; }
    const int l = m->level[ia];
    if (l >= nlv) { r->err = r->err ? r->err : 2; continue; }
    double Twa[7], Tla[7], x[3];
    oloop_se3_inv(m->pose + 7 * a, Twa);
    oloop_se3_mul(r->T_loop_from_w, Twa, Tla);
    oloop_se3_act(Tla, m->xyz + 3 * p, x);
    const omatch_level *L = &cur->levels[l];
    const double u = L->f * (x[0] / x[2]) + L->px, v = L->f * (x[1] / x[2]) + L->py;
    const int ui = (int)u, vi = (int)v;
    if (!(ui >= 0 && ui < L->w && vi >= 0 && vi < L->h)) continue;
    if (vertex_slot[a] < 0) { r->err = r->err ? r->err : 3; continue; }
    omatch_point *c = &pts[nc];
    c->keyframe = vertex_slot[a];
    c->anchor_level = l;
    const double s = (double)(1 << l);
    c->anchor_obs_pyr[0] = m->center[3 * ia] / s;
    c->anchor_obs_pyr[1] = m->center[3 * ia + 1] / s;
    memcpy(c->xyz_anchor, m->xyz + 3 * p, sizeof(double) * 3);
    cp[nc++] = p;
  }
  r->n_candidates = nc;
  if (cand_point) memcpy(cand_point, cp, sizeof(int) * nc);
  if (cand) memcpy(cand, pts, sizeof(omatch_point) * nc);
  if (r->err) { r->stage = -1; goto out; }
  /* the vertex_table: every slot its vertex's map pose, loop's slot the prediction */
  for (int v = 0; v < m->V; ++v)
    if (vertex_slot[v] >= 0 && vertex_slot[v] < nkf)
      memcpy(kfs[vertex_slot[v]].T_me_from_w, v == loop ? r->T_loop_from_w : m->pose + 7 * v, sizeof(double) * 7);
  /* matchAndAlign (:726-784) */
  double T[7] = {0, 0, 0, 1, 0, 0, 0};
  omatch_match(cur, kfs, nkf, T, r->T_loop_from_w, pts, nc, 10, 22, 10, ra);
  for (int i = 0; i < nc; ++i) r->n_matched1 += ra[i].matched;
  if (res1) memcpy(res1, ra, sizeof(omatch_result) * nc);
  if (r->n_matched1 < covis_thr) { r->stage = 1; goto out; }
  if (align(nc, ra, cam, 25, T, &r->lm[0])) { r->stage = -2; goto out; }
  memcpy(r->T_align1, T, sizeof T);
  omatch_match(cur, kfs, nkf, T, r->T_loop_from_w, pts, nc, 4, 22, 10, rb);
  for (int i = 0; i < nc; ++i) r->n_matched2 += rb[i].matched;
  if (res2) memcpy(res2, rb, sizeof(omatch_result) * nc);
  if (align(nc, rb, cam, 15, T, &r->lm[1])) { r->stage = -2; goto out; }
  memcpy(r->T_newloop_from_oldloop, T, sizeof T);
  if (r->n_matched2 < covis_thr) { r->stage = 2; goto out; }
  /* :904-961 */
  int nt = 0;
  const double w0 = cur->levels[0].w, h0 = cur->levels[0].h;
  for (int i = 0; i < nc; ++i) {
    if (!rb[i].matched) continue;
    double pred[3];
    oloop_map_uvu(cam, T, rb[i].xyz_actkey, pred);
    const double *uvu = rb[i].obs;
    const double d0 = uvu[0] - pred[0], d1 = uvu[1] - pred[1], d2 = uvu[2] - pred[2];
    const int factor = 1 << pts[i].anchor_level;
    if (fabs(d0) < 2.0 * factor && fabs(d1) < 2.0 * factor && fabs(d2) < 2.0 * 3) {
      if (uvu[0] > w0 * 0.5) r->num_right++; else r->num_left++;
      if (uvu[1] > h0 * 0.5) r->num_lower++; else r->num_upper++;
      if (track_point) { track_point[nt] = cp[i]; track_level[nt] = pts[i].anchor_level; memcpy(track_uvu + 3 * nt, uvu, sizeof(double) * 3); }
      ++nt;
    }
  }
  r->n_tracks = nt;
  if (nt < covis_thr) { r->stage = 3; goto out; }
  const int half = covis_thr / 2;
  if (r->num_lower < half || r->num_upper < half || r->num_left < half || r->num_right < half) { r->stage = 4; goto out; }
  /* :964-971 */
  double A[7];
  oloop_se3_mul(T, Tlq, A);
  oloop_se3_mul(A, m->pose + 7 * query, r->T_newloop_from_w);
  r->verified = 1;
  /* addNewObsToOldPoints on v_loop: feature_table.insert keeps an existing observation; vis_set in ascending order */
  if (vis_ptr2) {
    int *add = malloc(sizeof(int) * cap);
    for (int p = 0; p < m->Np; ++p) add[p] = -1;
    for (int t = 0; t < nt; ++t) add[track_point[t]] = t;
    int at = 0;
    for (int p = 0; p < m->Np; ++p) {
      vis_ptr2[p] = at;
      int t = add[p];
      for (int k = m->vis_ptr[p]; k < m->vis_ptr[p + 1]; ++k)
        if (m->vis_pose[k] == loop) t = -1;
      for (int k = m->vis_ptr[p]; k <= m->vis_ptr[p + 1]; ++k) {
        if (t >= 0 && (k == m->vis_ptr[p + 1] || m->vis_pose[k] > loop)) {
          vis_pose2[at] = loop; level2[at] = track_level[t]; memcpy(center2 + 3 * at, track_uvu + 3 * t, sizeof(double) * 3);
          ++at; t = -1;
        }
        if (k == m->vis_ptr[p + 1]) break;
        vis_pose2[at] = m->vis_pose[k]; level2[at] = m->level[k]; memcpy(center2 + 3 * at, m->center + 3 * k, sizeof(double) * 3);
        ++at;
      }
    }
    vis_ptr2[m->Np] = at;
    r->nnz2 = at;
    free(add);
  }
out:
  free(inwin); free(cp); free(pts); free(ra); free(rb);
}
