/* prepare_oracle.c -- see prepare_oracle.h.  TEST INFRASTRUCTURE ONLY.  PARITY UNPINNED. */
#include "prepare_oracle.h"

#include <stdlib.h>
#include <string.h>

#include "ba_oracle.h"
#include "constraint_oracle.h"

/* EdgeTable: the undirected edges (id1 < id2) in ascending order, found by bisection (orderd_find) */
typedef struct { int n; long long *key; double *T, *L12, *L21; unsigned char *mrg, *rew; } OEdges;

static int oedge_find(const OEdges *e, int a, int b) {
  const long long k = a < b ? (long long)a << 32 | (unsigned)b : (long long)b << 32 | (unsigned)a;
  int lo = 0, hi = e->n;
  while (lo < hi) { const int mid = (lo + hi) / 2; if (e->key[mid] < k) lo = mid + 1; else hi = mid; }
  return lo < e->n && e->key[lo] == k ? lo : -1;
}

static int cmp_ll(const void *a, const void *b) {
  const long long x = *(const long long *)a, y = *(const long long *)b;
  return x < y ? -1 : x > y;
}

/* getRelativePose_1_from_2 (slam_graph.cpp:271-286) with getConstraint_id1_from_id2 (slam_graph.hpp:242-287) */
static void orel_pose(const OEdges *e, const double *poses, int id1, int id2, double *T12) {
  const int k = oedge_find(e, id1, id2);
  if (e->mrg[k]) {
    if (id1 < id2) memcpy(T12, e->T + 7 * k, sizeof(double) * 7);
    else oba_se3_inv(e->T + 7 * k, T12);
    return;
  }
  double inv2[7];
  oba_se3_inv(poses + 7 * id2, inv2);
  oba_se3_mul(poses + 7 * id1, inv2, T12);
}

/* EdgeTable::setConstraint (slam_graph.hpp:295-331) */
static void oset_constraint(OEdges *e, int id1, int id2, const double *T12, const double *L12, const double *L21) {
  const int k = oedge_find(e, id1, id2);
  e->mrg[k] = 1; e->rew[k] = 1;
  if (id1 < id2) {
    memcpy(e->T + 7 * k, T12, sizeof(double) * 7);
    memcpy(e->L21 + 36 * k, L21, sizeof(double) * 36); memcpy(e->L12 + 36 * k, L12, sizeof(double) * 36);
  } else {
    oba_se3_inv(T12, e->T + 7 * k);
    memcpy(e->L21 + 36 * k, L12, sizeof(double) * 36); memcpy(e->L12 + 36 * k, L21, sizeof(double) * 36);
  }
}

typedef struct { int own_id, parent_id; double T_parent_from_world[7]; int mark_reinitialize; } ReinitializeTraversalNode;

void opr_prepare_for_optimization(int V, const int *nbr_ptr, const int *nbr_id, const double *nbr_T, const double *nbr_L,
                                  const unsigned char *nbr_mrg, const int *old_type, const int *new_type, int root, int loop,
                                  double *poses, const int *feat_ptr, const int *feat_point, int Np, const int *point_anchor,
                                  const double *xyz_anchor, double *out_T, double *out_L, unsigned char *out_mrg,
                                  unsigned char *rewritten) {
  const int nn = nbr_ptr[V];
  OEdges e = {0};
  e.key = malloc(sizeof(long long) * (size_t)(nn + 1));
  for (int v = 0; v < V; ++v)
    for (int i = nbr_ptr[v]; i < nbr_ptr[v + 1]; ++i)
      if (v < nbr_id[i]) e.key[e.n++] = (long long)v << 32 | (unsigned)nbr_id[i];
  qsort(e.key, (size_t)e.n, sizeof(long long), cmp_ll);
  e.T = malloc(sizeof(double) * 7 * (size_t)(e.n + 1));
  e.L12 = malloc(sizeof(double) * 36 * (size_t)(e.n + 1)); e.L21 = malloc(sizeof(double) * 36 * (size_t)(e.n + 1));
  e.mrg = calloc((size_t)e.n + 1, 1); e.rew = calloc((size_t)e.n + 1, 1);
  for (int v = 0; v < V; ++v)   /* entry (me -> nbr) holds T_nbr_from_me: the max -> min entry is T_1_from_2 (1 = min) */
    for (int i = nbr_ptr[v]; i < nbr_ptr[v + 1]; ++i) {
      const int b = nbr_id[i], k = oedge_find(&e, v, b);
      if (v > b) { memcpy(e.T + 7 * k, nbr_T + 7 * i, sizeof(double) * 7); memcpy(e.L12 + 36 * k, nbr_L + 36 * i, sizeof(double) * 36); e.mrg[k] = nbr_mrg[i]; }
      else memcpy(e.L21 + 36 * k, nbr_L + 36 * i, sizeof(double) * 36);
    }
  /* reinitializePoses: queue<ReinitializeTraversalNode>, cycle_check */
  ReinitializeTraversalNode *queue = malloc(sizeof(ReinitializeTraversalNode) * (size_t)(nn + 1));
  unsigned char *cycle_check = calloc((size_t)V, 1);
  int head = 0, tail = 0;
  queue[tail].own_id = root; queue[tail].parent_id = -1; queue[tail].mark_reinitialize = 0;
  memcpy(queue[tail].T_parent_from_world, (const double[7]){0, 0, 0, 1, 0, 0, 0}, sizeof(double) * 7);
  ++tail;
  while (head < tail) {
    const ReinitializeTraversalNode node = queue[head++];
    if (cycle_check[node.own_id]) continue;          /* Avoid cycles! */
    if (new_type[node.own_id] == 0) continue;        /* Skip is it is not in double window */
    cycle_check[node.own_id] = 1;
    const int reinitialize_me_and_my_childs = node.mark_reinitialize || node.own_id == loop;
    if (node.parent_id > -1 && (reinitialize_me_and_my_childs || old_type[node.own_id] == 0)) {
      double rel[7];
      orel_pose(&e, poses, node.own_id, node.parent_id, rel);
      oba_se3_mul(rel, node.T_parent_from_world, poses + 7 * node.own_id);
    }
    for (int i = nbr_ptr[node.own_id]; i < nbr_ptr[node.own_id + 1]; ++i) {   /* rbegin: strongest first */
      queue[tail].own_id = nbr_id[i]; queue[tail].parent_id = node.own_id;
      memcpy(queue[tail].T_parent_from_world, poses + 7 * node.own_id, sizeof(double) * 7);
      queue[tail].mark_reinitialize = reinitialize_me_and_my_childs;
      ++tail;
    }
  }
  int size = 0;
  for (int v = 0; v < V; ++v) size += new_type[v] != 0;
  if (size >= 2) {
    /* unmargPosesEnteringInnerW */
    for (int id1 = 0; id1 < V; ++id1) {
      if (new_type[id1] != 1) continue;
      for (int id2 = 0; id2 < V; ++id2) {
        if (!new_type[id2] || id2 == id1) continue;
        if (new_type[id2] == 1) {
          const int k = oedge_find(&e, id1, id2);
          if (k >= 0) e.mrg[k] = 0;
        }
      }
    }
    /* margPosesLeftInnerWindow(old_window) */
    for (int id1 = 0; id1 < V; ++id1) {
      if (old_type[id1] != 1) continue;
      for (int id2 = 0; id2 < V; ++id2) {
        if (!old_type[id2] || id2 == id1) continue;
        if (oedge_find(&e, id1, id2) < 0) continue;
        if (old_type[id2] == 1 && !(new_type[id1] == 1 && new_type[id2] == 1)) {
          double T12[7], Lam[36];
          int vis;
          occ_compute_constraints(V, poses, feat_ptr, feat_point, Np, point_anchor, xyz_anchor, 1, &id1, &id2, T12, Lam, &vis);
          oset_constraint(&e, id1, id2, T12, Lam, Lam);
        }
      }
    }
  }
  for (int v = 0; v < V; ++v)
    for (int i = nbr_ptr[v]; i < nbr_ptr[v + 1]; ++i) {
      const int b = nbr_id[i], k = oedge_find(&e, v, b);
      out_mrg[i] = e.mrg[k]; rewritten[i] = e.rew[k];
      if (!e.rew[k]) {
        memcpy(out_T + 7 * i, nbr_T + 7 * i, sizeof(double) * 7); memcpy(out_L + 36 * i, nbr_L + 36 * i, sizeof(double) * 36);
      } else if (b < v) {          /* getConstraint_id1_from_id2(b, v) with b < v */
        memcpy(out_T + 7 * i, e.T + 7 * k, sizeof(double) * 7); memcpy(out_L + 36 * i, e.L12 + 36 * k, sizeof(double) * 36);
      } else {
        oba_se3_inv(e.T + 7 * k, out_T + 7 * i); memcpy(out_L + 36 * i, e.L21 + 36 * k, sizeof(double) * 36);
      }
    }
  free(e.key); free(e.T); free(e.L12); free(e.L21); free(e.mrg); free(e.rew); free(queue); free(cycle_check);
}
