/* register_oracle.c -- see register_oracle.h.  TEST INFRASTRUCTURE ONLY.  Written sequentially from backend.cpp:433-784
 * and slam_graph.cpp:105-140, 189-205, 400-420; the projections are restated operation by operation without FMA
 * contraction (the pragma keeps it so under the Makefile's flags), like csrc/loop.cu compiled with -fmad=false. */
#pragma GCC optimize("fp-contract=off")
#include "register_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

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

static int observes(const oloop_map *m, int p, int v) {
  for (int k = m->vis_ptr[p]; k < m->vis_ptr[p + 1]; ++k)
    if (m->vis_pose[k] == v) return 1;
  return 0;
}

void oreg_local_register_frame(const oloop_map *m, const int *nbr_ptr, const int *nbr_id, const omatch_frame *cur,
                               omatch_keyframe *kfs, int nkf, const double cam[4], int covis_thr, int root, int P,
                               const int *window_vertex, const int *vertex_slot, oreg_result *r, int *direct_out,
                               int *neighborhood_out, int *cand_point, omatch_point *cand, omatch_result *res1,
                               omatch_result *res2, oreg_stats *stats, int *track_point, double *track_uvu,
                               int *track_level, int *track_committed, int *vis_ptr2, int *vis_pose2, double *center2,
                               int *level2) {
  memset(r, 0, sizeof *r);
  const int V = m->V;
  int nlv = 0;
  while (nlv < OMATCH_MAX_LEVELS && cur->levels[nlv].w > 0) ++nlv;
  char *inwin = calloc((size_t)V, 1), *direct = calloc((size_t)V, 1), *larger = calloc((size_t)V, 1);
  char *anch = calloc((size_t)V, 1), *qual = calloc((size_t)V, 1);
  for (int i = 0; i < P; ++i) inwin[window_vertex[i]] = 1;
  const int cap = m->Np > 0 ? m->Np : 1;
  int *cp = malloc(sizeof(int) * cap), *kept = malloc(sizeof(int) * cap);
  omatch_point *pts = malloc(sizeof(omatch_point) * cap);
  omatch_result *ra = malloc(sizeof(omatch_result) * cap), *rb = malloc(sizeof(omatch_result) * cap);
  int *cnt = calloc((size_t)V * 5, sizeof(int));
  int *queue = malloc(sizeof(int) * ((size_t)nbr_ptr[V] + 1));
  char *seen = calloc((size_t)cap, 1);
  /* directNeighborsOf (:433-449) */
  direct[root] = 1;
  r->n_direct = 1;
  for (int i = nbr_ptr[root]; i < nbr_ptr[root + 1]; ++i)
    if (!direct[nbr_id[i]]) { direct[nbr_id[i]] = 1; r->n_direct++; }
  /* framesInNeighborhood(root, |direct| + 40) (slam_graph.cpp:105-140) */
  {
    const int size = r->n_direct + 40;
    int head = 0, tail = 0;
    queue[tail++] = root;
    while (tail != head && r->n_neighborhood < size) {
      const int v = queue[head++];
      if (larger[v]) continue;                                  /* Avoid cycles! */
      if (!inwin[v]) continue;
      larger[v] = 1;
      r->n_neighborhood++;
      for (int i = nbr_ptr[v]; i < nbr_ptr[v + 1]; ++i) queue[tail++] = nbr_id[i];   /* rbegin: strongest first */
    }
  }
  if (direct_out) for (int v = 0; v < V; ++v) direct_out[v] = direct[v];
  if (neighborhood_out) for (int v = 0; v < V; ++v) neighborhood_out[v] = larger[v];
  /* pointsVisibleInRoot (:472-546), the points in ascending index */
  for (int p = 0; p < m->Np; ++p)
    for (int k = m->vis_ptr[p]; k < m->vis_ptr[p + 1]; ++k)
      if (larger[m->vis_pose[k]] && !direct[m->vis_pose[k]]) seen[p] = 1;
  const double *Trw = m->pose + 7 * root;
  int nc = 0;
  for (int p = 0; p < m->Np; ++p) {
    if (!seen[p]) continue;
    const int a = m->anchor[p];
    if (!inwin[a]) continue;
    int ia = -1;
    for (int k = m->vis_ptr[p]; k < m->vis_ptr[p + 1] && ia < 0; ++k)
      if (m->vis_pose[k] == a) ia = k;
    if (ia < 0) { r->err = 1; continue; }
    const int l = m->level[ia];
    if (l >= nlv) { r->err = r->err ? r->err : 2; continue; }
    double Twa[7], Tra[7], x[3];
    oloop_se3_inv(m->pose + 7 * a, Twa);
    oloop_se3_mul(Trw, Twa, Tra);
    oloop_se3_act(Tra, m->xyz + 3 * p, x);
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
    anch[a] = 1;                                                /* vertex_table */
    cp[nc++] = p;
  }
  r->n_candidates = nc;
  if (cand_point) memcpy(cand_point, cp, sizeof(int) * nc);
  if (cand) memcpy(cand, pts, sizeof(omatch_point) * nc);
  if (r->err) { r->stage = -1; goto out; }
  if (nc < covis_thr) { r->stage = 1; goto out; }
  /* the vertex_table: every slot its vertex's map pose */
  for (int v = 0; v < V; ++v)
    if (vertex_slot[v] >= 0 && vertex_slot[v] < nkf) memcpy(kfs[vertex_slot[v]].T_me_from_w, m->pose + 7 * v, sizeof(double) * 7);
  /* matchAndAlign (:725-784) */
  double T[7] = {0, 0, 0, 1, 0, 0, 0};
  omatch_match(cur, kfs, nkf, T, Trw, pts, nc, 10, 22, 10, ra);
  for (int i = 0; i < nc; ++i) r->n_matched1 += ra[i].matched;
  if (res1) memcpy(res1, ra, sizeof(omatch_result) * nc);
  if (r->n_matched1 < covis_thr) { r->stage = 2; goto out; }
  if (align(nc, ra, cam, 25, T, &r->lm[0])) { r->stage = -2; goto out; }
  memcpy(r->T_align1, T, sizeof T);
  omatch_match(cur, kfs, nkf, T, Trw, pts, nc, 4, 22, 10, rb);
  for (int i = 0; i < nc; ++i) r->n_matched2 += rb[i].matched;
  if (res2) memcpy(res2, rb, sizeof(omatch_result) * nc);
  if (align(nc, rb, cam, 15, T, &r->lm[1])) { r->stage = -2; goto out; }
  memcpy(r->T_newroot_from_oldroot, T, sizeof T);
  if (r->n_matched2 < covis_thr) { r->stage = 3; goto out; }
  /* keyframesToRegister (:615-722) */
  const double w0 = cur->levels[0].w, h0 = cur->levels[0].h;
  int nt = 0;
  for (int i = 0; i < nc; ++i) {
    if (!rb[i].matched) continue;
    double pred[3];
    oloop_map_uvu(cam, T, rb[i].xyz_actkey, pred);
    const double *uvu = rb[i].obs;
    const double d0 = uvu[0] - pred[0], d1 = uvu[1] - pred[1], d2 = uvu[2] - pred[2];
    const int factor = 1 << pts[i].anchor_level;
    if (!(fabs(d0) < 2.0 * factor && fabs(d1) < 2.0 * factor && fabs(d2) < 2.0 * 3)) continue;
    kept[nt] = cp[i];
    if (track_point) { track_point[nt] = cp[i]; track_level[nt] = pts[i].anchor_level; memcpy(track_uvu + 3 * nt, uvu, sizeof(double) * 3); }
    ++nt;
    for (int v = 0; v < V; ++v) {                               /* vertex_table = root and the anchors */
      if ((!anch[v] && v != root) || direct[v] || !observes(m, cp[i], v)) continue;
      int *c = cnt + 5 * v;
      c[0]++;                                                   /* point_list.size() */
      if (uvu[0] > w0 * 0.5) c[1]++; else c[2]++;               /* num_left, num_right as the reference names them */
      if (uvu[1] > h0 * 0.5) c[4]++; else c[3]++;               /* num_lower, num_upper */
    }
  }
  r->n_tracks = nt;
  const int half = covis_thr / 2;
  for (int v = 0; v < V; ++v) {
    const int *c = cnt + 5 * v;
    if (c[0] == 0) continue;
    qual[v] = c[0] >= covis_thr && c[1] >= half && c[2] >= half && c[3] >= half && c[4] >= half;
    if (stats) { oreg_stats s = {v, c[0], c[1], c[2], c[3], c[4], qual[v]}; stats[r->n_stats] = s; }
    r->n_stats++;
    r->n_neighbors += qual[v];
  }
  int *add = malloc(sizeof(int) * cap);
  for (int p = 0; p < m->Np; ++p) add[p] = -1;
  for (int t = 0; t < nt; ++t) {
    int com = 0;
    for (int v = 0; v < V; ++v) com |= qual[v] && observes(m, kept[t], v);
    if (track_committed) track_committed[t] = com;
    if (com) { add[kept[t]] = t; r->n_committed++; }
  }
  if (r->n_neighbors == 0) { r->stage = 4; free(add); goto out; }
  oloop_se3_mul(T, Trw, r->T_newroot_from_w);
  r->registered = 1;
  /* registerKeyframes: addNewObsToOldPoints on v_root, feature_table.insert keeps an existing observation */
  if (vis_ptr2) {
    int at = 0;
    for (int p = 0; p < m->Np; ++p) {
      vis_ptr2[p] = at;
      int t = add[p];
      if (observes(m, p, root)) t = -1;
      for (int k = m->vis_ptr[p]; k <= m->vis_ptr[p + 1]; ++k) {
        if (t >= 0 && (k == m->vis_ptr[p + 1] || m->vis_pose[k] > root)) {
          vis_pose2[at] = root; level2[at] = track_level[t]; memcpy(center2 + 3 * at, track_uvu + 3 * t, sizeof(double) * 3);
          ++at; t = -1;
        }
        if (k == m->vis_ptr[p + 1]) break;
        vis_pose2[at] = m->vis_pose[k]; level2[at] = m->level[k]; memcpy(center2 + 3 * at, m->center + 3 * k, sizeof(double) * 3);
        ++at;
      }
    }
    vis_ptr2[m->Np] = at;
    r->nnz2 = at;
  }
  free(add);
out:
  free(inwin); free(direct); free(larger); free(anch); free(qual); free(cp); free(kept); free(pts); free(ra); free(rb);
  free(cnt); free(queue); free(seen);
}
