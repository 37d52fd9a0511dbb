/* frontend_oracle.c -- see frontend_oracle.h.  TEST INFRASTRUCTURE ONLY.  Written sequentially from
 * stereo_frontend.cpp:512-528, :724-823, :834-974 and :977-1065; the projections are restated operation by operation
 * without FMA contraction (the pragma keeps it so under the Makefile's flags), like csrc/frontend_points.cu compiled
 * with -fmad=false.  The window test is the literal cv::Rect_<double>::contains over every point of the tree, and the
 * seeding's greedy runs one corner after the other in emission order. */
#pragma GCC optimize("fp-contract=off")
#include "frontend_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "loop_oracle.h"

void ofront_budget(omatch_result *res, int n_groups, const int *group_end, int num_max_points, int *num_new,
                   int *num_obs) {
  int total = 0, keep = 1;
  *num_new = 0;
  for (int g = 0; g < n_groups; ++g) {
    const int b0 = g ? group_end[g - 1] : 0, b1 = group_end[g];
    const int neighbour = g > 0 && g < n_groups - 1;
    if (neighbour) keep = keep && 2 * total < num_max_points;   /* the for condition of :1007-1010 */
    for (int i = b0; i < b1; ++i) {
      if (neighbour && !keep) res[i].matched = 0;
      total += res[i].matched;
    }
    if (g == n_groups - 2) *num_new = total;
  }
  *num_obs = total;
}

static void thirds(int w, int *t, int *tt) {
  const float third = (float)(1. / 3.);
  *t = (int)((float)w * third);
  *tt = (int)((float)(w * 2) * third);
}

int ofront_process(const omatch_result *res, const int *anchor_level, int n, int n_new, const double T[7],
                   const double cam[4], int w0, int h0, float max_err, int min_num_points, ofront_tracked *out,
                   ofront_stats *st, int flags[9]) {
  memset(st, 0, sizeof *st);
  const int half_w = (int)(w0 * 0.5), half_h = (int)(h0 * 0.5);
  int tw, ttw, th, tth;
  thirds(w0, &tw, &ttw);
  thirds(h0, &th, &tth);
  double sum = 0.;
  int cnt = 0;
  for (int i = 0; i < n; ++i) {
    if (!res[i].matched) continue;
    const int lvl = anchor_level[i];
    double pred[3];
    oloop_map_uvu(cam, T, res[i].xyz_actkey, pred);
    const double d0 = res[i].obs[0] - pred[0], d1 = res[i].obs[1] - pred[1], d2 = res[i].obs[2] - pred[2];
    const int factor = 1 << lvl;
    if (!(fabs(d0) < max_err * factor && fabs(d1) < max_err * factor && fabs(d2) < 3. * max_err)) continue;
    const double *uvu = res[i].obs;
    ++st->grid2x2[uvu[0] < half_w ? 0 : 1][uvu[1] < half_h ? 0 : 1];
    ++st->grid3x3[uvu[0] < tw ? 0 : (uvu[0] < ttw ? 1 : 2)][uvu[1] < th ? 0 : (uvu[1] < tth ? 1 : 2)];
    ++st->num_matched_points[lvl];
    const double s = (double)factor;
    const double *X = res[i].xyz_actkey;
    const double cu = (cam[0] * (X[0] / X[2]) + cam[1]) / s, cv = (cam[0] * (X[1] / X[2]) + cam[2]) / s;
    const double du = uvu[0] / s - cu, dv = uvu[1] / s - cv;
    sum += sqrt(du * du + dv * dv);
    ofront_tracked *o = out + cnt;
    o->index = i; o->is_new = i < n_new; o->anchor_level = lvl; o->reserved = 0;
    o->uvu[0] = uvu[0]; o->uvu[1] = uvu[1]; o->uvu[2] = uvu[2];
    st->num_new += i < n_new;
    ++cnt;
  }
  st->num_tracked = cnt;
  st->av_track_length = sum / cnt;
  for (int k = 0; k < 9; ++k) flags[k] = st->grid3x3[k / 3][k % 3] <= min_num_points;
  return cnt;
}

int ofront_drop(const ofront_stats *st, const double T[7], int featureless_corners_thr, float parallax_thr) {
  int featureless = 0;
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j)
      if (st->grid2x2[i][j] < 15) ++featureless;
  const double tn = sqrt(T[4] * T[4] + T[5] * T[5] + T[6] * T[6]);
  return featureless > featureless_corners_thr || tn > parallax_thr || st->av_track_length > 75.;
}

static unsigned long long sm64(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ull;
  unsigned long long z = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
unsigned long long ofront_hash5(unsigned long long a, unsigned long long b, unsigned long long c, unsigned long long d,
                                unsigned long long e) {
  return sm64(sm64(sm64(sm64(sm64(a) ^ b) ^ c) ^ d) ^ e);
}

#define DEPTH 16

/* the node path of (u, v) at depth d of the regular midpoint tree over [0, w) x [0, h) */
static unsigned long long node_path(int w, int h, int u, int v, int d) {
  double x = 0, y = 0, ww = w, hh = h;
  unsigned long long P = 0;
  for (int k = 0; k < d; ++k) {
    const double x1 = x + ww * 0.5, y1 = y + hh * 0.5;
    const int bx = u >= x1, by = v >= y1;
    if (bx) x = x1;
    if (by) y = y1;
    ww = ww * 0.5; hh = hh * 0.5;
    P = (P << 2) | (unsigned long long)((bx << 1) | by);
  }
  return P;
}

typedef struct { unsigned long long h, path; int c; } emit_rec;
static int emit_cmp(const void *pa, const void *pb) {
  const emit_rec *a = pa, *b = pb;
  if (a->h != b->h) return a->h < b->h ? -1 : 1;
  if (a->path != b->path) return a->path < b->path ? -1 : 1;
  return 0;
}
/* corners sorted by full-depth path, then index: the nodes of every depth are runs of this order */
static const unsigned long long *g_full;
static int full_cmp(const void *pa, const void *pb) {
  const int a = *(const int *)pa, b = *(const int *)pb;
  if (g_full[a] != g_full[b]) return g_full[a] < g_full[b] ? -1 : 1;
  return a < b ? -1 : (a > b);
}

int ofront_emission_order(int w, int h, int level, const int *xy, int n, unsigned long long seed, int *order) {
  const int n1 = n ? n : 1;
  int *alive = malloc(sizeof(int) * n1), *srt = malloc(sizeof(int) * n1);
  unsigned long long *key = malloc(sizeof(unsigned long long) * n1), *full = malloc(sizeof(unsigned long long) * n1);
  emit_rec *rec = malloc(sizeof(emit_rec) * n1);
  for (int i = 0; i < n; ++i) {
    key[i] = ofront_hash5(seed, 0, (unsigned long long)level, (unsigned long long)xy[2 * i], (unsigned long long)xy[2 * i + 1]);
    full[i] = node_path(w, h, xy[2 * i], xy[2 * i + 1], DEPTH);
    srt[i] = i;
  }
  g_full = full;
  qsort(srt, n, sizeof(int), full_cmp);
  /* of corners at one position (one full-depth node) only the lowest index exists */
  for (int k = 0; k < n; ++k) alive[srt[k]] = !(k > 0 && full[srt[k - 1]] == full[srt[k]]);
  int m = 0;
  for (int d = 0; d <= DEPTH; ++d) {
    /* every node holding a corner not yet emitted emits the smallest (key, index) */
    const int sh = 2 * (DEPTH - d);
    int nr = 0;
    for (int k0 = 0; k0 < n;) {
      int k1 = k0 + 1;
      while (k1 < n && (full[srt[k1]] >> sh) == (full[srt[k0]] >> sh)) ++k1;
      int best = -1;
      for (int k = k0; k < k1; ++k) {
        const int c = srt[k];
        if (alive[c] != 1) continue;
        if (best < 0 || key[c] < key[best] || (key[c] == key[best] && c < best)) best = c;
      }
      if (best >= 0) {
        rec[nr].h = ofront_hash5(seed, 1, (unsigned long long)level, (unsigned long long)d, full[best] >> sh);
        rec[nr].path = full[best] >> sh;
        rec[nr].c = best;
        ++nr;
      }
      k0 = k1;
    }
    qsort(rec, nr, sizeof *rec, emit_cmp);
    for (int k = 0; k < nr; ++k) { order[m++] = rec[k].c; alive[rec[k].c] = 2; }
  }
  free(alive); free(srt); free(key); free(full); free(rec);
  return m;
}

static int rect_contains(double cx, double cy, int R, double px, double py) {
  const double x = cx - R, y = cy - R, d = 2 * R + 1;
  return x <= px && px < x + d && y <= py && py < y + d;
}

int ofront_seed(int nlevels, const int *w, const int *h, const int *const *xy, const int *nkp, const float *disp,
                int disp_pitch, const ofront_tracked *tree, int ntrk, const int *num_in, const int flags[9], int R,
                int num_max_points, unsigned long long seed, const double T[7], const double cam[4], int slot,
                ofront_new_point *points, omatch_point *rows, int *counts) {
  const int w0 = w[0], h0 = h[0];
  int tw, ttw, th, tth;
  thirds(w0, &tw, &ttw);
  thirds(h0, &th, &tth);
  int total = 0;
  for (int l = 0; l < nlevels; ++l) {
    const double sl = (double)(1 << l), inv_factor = 1. / (double)(1 << l);
    /* the level's tree: the gated points at uv_pyr, then the taken corners */
    double *tp = malloc(sizeof(double) * 2 * (size_t)(ntrk + nkp[l] + 1));
    int nt = 0;
    for (int k = 0; k < ntrk; ++k)
      if (tree[k].anchor_level == l) { tp[2 * nt] = tree[k].uvu[0] / sl; tp[2 * nt + 1] = tree[k].uvu[1] / sl; ++nt; }
    int *order = malloc(sizeof(int) * (size_t)(nkp[l] ? nkp[l] : 1));
    const int m = ofront_emission_order(w[l], h[l], l, xy[l], nkp[l], seed, order);
    const int cap = num_max_points >> l;
    int num = num_in[l], kept = 0;
    for (int k = 0; k < m; ++k) {
      const int c = order[k];
      const int u = xy[l][2 * c], v = xy[l][2 * c + 1];
      const int uz = u << l, vz = v << l;
      const double dsp = uz < w0 && vz < h0 ? (double)disp[(size_t)vz * disp_pitch + uz] * inv_factor : 0.;
      if (!(dsp > 0)) continue;
      if (!(uz >= 1 && uz < w0 - 1 && vz >= 1 && vz < h0 - 1)) continue;
      if (!flags[(uz < tw ? 0 : (uz < ttw ? 1 : 2)) * 3 + (vz < th ? 0 : (vz < tth ? 1 : 2))]) continue;
      int empty = 1;
      for (int q = 0; q < nt && empty; ++q)
        if (rect_contains(u, v, R, tp[2 * q], tp[2 * q + 1])) empty = 0;
      if (!empty) continue;
      tp[2 * nt] = u; tp[2 * nt + 1] = v; ++nt;
      ofront_new_point *p = points + total;
      p->level = l; p->reserved = 0;
      p->uv_pyr[0] = u; p->uv_pyr[1] = v;
      p->uvu_pyr[0] = u; p->uvu_pyr[1] = v; p->uvu_pyr[2] = u - dsp;
      const double u0 = p->uvu_pyr[0] * sl, v0 = p->uvu_pyr[1] * sl, r0 = p->uvu_pyr[2] * sl;
      const double sd = (u0 - r0) / cam[3];
      const double z = cam[0] / sd;
      const double xc[3] = {(u0 - cam[1]) / cam[0] * z, (v0 - cam[2]) / cam[0] * z, z};
      oloop_se3_act(T, xc, p->xyz);
      const double dist = sqrt(xc[0] * xc[0] + xc[1] * xc[1] + xc[2] * xc[2]);
      for (int q = 0; q < 3; ++q) p->normal[q] = -xc[q] / dist;
      omatch_point *r = rows + total;
      r->keyframe = slot; r->anchor_level = l;
      for (int q = 0; q < 3; ++q) r->xyz_anchor[q] = p->xyz[q];
      r->anchor_obs_pyr[0] = u; r->anchor_obs_pyr[1] = v;
      ++total; ++kept;
      ++num;
      if (num > cap) break;
    }
    counts[l] = kept;
    free(tp); free(order);
  }
  return total;
}
