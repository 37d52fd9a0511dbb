/* graph_oracle.c -- see graph_oracle.h.  TEST INFRASTRUCTURE ONLY.  PARITY UNPINNED. */
#include "graph_oracle.h"

#include <stdlib.h>
#include <string.h>

#include "ba_oracle.h"
#include "constraint_oracle.h"

void ogr_compute_strength(int V, const int *vis_ptr, const int *vis_pose, int n_new, const int *new_anchor, int n_track,
                          const int *track_point, const double *track_center, int covis_thr, int width, int height,
                          int *in_table, int *strength) {
  /* IntTable as arrays over the vertices, IS_IN_SET as a presence flag per table */
  int *top = calloc((size_t)V, sizeof(int)), *bottom = calloc((size_t)V, sizeof(int));
  int *left = calloc((size_t)V, sizeof(int)), *right = calloc((size_t)V, sizeof(int));
  unsigned char *in_t = calloc((size_t)V, 1), *in_b = calloc((size_t)V, 1), *in_l = calloc((size_t)V, 1), *in_r = calloc((size_t)V, 1);
  memset(in_table, 0, sizeof(int) * (size_t)V);
  memset(strength, 0, sizeof(int) * (size_t)V);
  const int half_width = width * 0.5, half_height = height * 0.5;
  for (int q = 0; q < n_new; ++q) { in_table[new_anchor[q]] = 1; strength[new_anchor[q]] += 1; }
  for (int t = 0; t < n_track; ++t) {
    const int p = track_point[t];
    for (int i = vis_ptr[p]; i < vis_ptr[p + 1]; ++i) {
      const int f = vis_pose[i];
      in_table[f] = 1; strength[f] += 1;
      const double u = track_center[3 * t], v = track_center[3 * t + 1];
      if (u < half_width) { in_l[f] = 1; left[f] += 1; } else { in_r[f] = 1; right[f] += 1; }
      if (v < half_height) { in_t[f] = 1; top[f] += 1; } else { in_b[f] = 1; bottom[f] += 1; }
    }
    for (int f = 0; f < V; ++f) { /* the zeroing loop inside the track loop (:532-550) */
      if (!in_table[f]) continue;
      if (in_t[f] && top[f] >= covis_thr / 2 && in_b[f] && bottom[f] >= covis_thr / 2 && in_l[f] && left[f] >= covis_thr / 2 &&
          in_r[f] && right[f] >= covis_thr / 2)
        continue;
      strength[f] = 0;
    }
  }
  free(top); free(bottom); free(left); free(right); free(in_t); free(in_b); free(in_l); free(in_r);
}

/* one neighbour list as the multimap holds it: ascending key, equal keys in insertion order */
typedef struct { int n, cap; int *key, *id; double *T, *L; } OList;

static void olist_insert(OList *l, int key, int id, const double *T, const double *L) {
  if (l->n == l->cap) {
    l->cap = l->cap ? 2 * l->cap : 8;
    l->key = realloc(l->key, sizeof(int) * (size_t)l->cap); l->id = realloc(l->id, sizeof(int) * (size_t)l->cap);
    l->T = realloc(l->T, sizeof(double) * 7 * (size_t)l->cap); l->L = realloc(l->L, sizeof(double) * 36 * (size_t)l->cap);
  }
  int at = l->n; /* upper bound: after every key <= key */
  while (at > 0 && l->key[at - 1] > key) --at;
  memmove(l->key + at + 1, l->key + at, sizeof(int) * (size_t)(l->n - at));
  memmove(l->id + at + 1, l->id + at, sizeof(int) * (size_t)(l->n - at));
  memmove(l->T + 7 * (at + 1), l->T + 7 * at, sizeof(double) * 7 * (size_t)(l->n - at));
  memmove(l->L + 36 * (at + 1), l->L + 36 * at, sizeof(double) * 36 * (size_t)(l->n - at));
  l->key[at] = key; l->id[at] = id;
  memcpy(l->T + 7 * at, T, sizeof(double) * 7); memcpy(l->L + 36 * at, L, sizeof(double) * 36);
  ++l->n;
}

void ogr_add_edges(int gV, int V, const int *nbr_ptr, const int *nbr_id, const int *nbr_str, const double *nbr_T,
                   const double *nbr_L, int n, const int *v1, const int *v2, const int *s, const double *poses,
                   const int *feat_ptr, const int *feat_point, int Np, const int *point_anchor, const double *xyz_anchor,
                   int *out_ptr, int *out_id, int *out_str, double *out_T, double *out_L) {
  OList *lists = calloc((size_t)V, sizeof(OList));
  for (int v = 0; v < gV; ++v) /* the stored lists are rbegin order: the multimap holds them reversed */
    for (int i = nbr_ptr[v + 1] - 1; i >= nbr_ptr[v]; --i) olist_insert(&lists[v], nbr_str[i], nbr_id[i], nbr_T + 7 * i, nbr_L + 36 * i);
  double *T12 = malloc(sizeof(double) * 7 * (size_t)(n + 1)), *Lam = malloc(sizeof(double) * 36 * (size_t)(n + 1));
  int *vis = malloc(sizeof(int) * (size_t)(n + 1));
  occ_compute_constraints(V, poses, feat_ptr, feat_point, Np, point_anchor, xyz_anchor, n, v1, v2, T12, Lam, vis);
  for (int k = 0; k < n; ++k) {
    double T21[7];
    oba_se3_inv(T12 + 7 * k, T21);
    olist_insert(&lists[v1[k]], s[k], v2[k], T21, Lam + 36 * k);        /* v1's entry for v2: T_2_from_1 */
    olist_insert(&lists[v2[k]], s[k], v1[k], T12 + 7 * k, Lam + 36 * k); /* v2's entry for v1: T_1_from_2 */
  }
  int at = 0;
  out_ptr[0] = 0;
  for (int v = 0; v < V; ++v) {
    OList *l = &lists[v];
    for (int i = l->n - 1; i >= 0; --i, ++at) {
      out_id[at] = l->id[i]; out_str[at] = l->key[i];
      memcpy(out_T + 7 * at, l->T + 7 * i, sizeof(double) * 7); memcpy(out_L + 36 * at, l->L + 36 * i, sizeof(double) * 36);
    }
    out_ptr[v + 1] = at;
    free(l->key); free(l->id); free(l->T); free(l->L);
  }
  free(lists); free(T12); free(Lam); free(vis);
}
