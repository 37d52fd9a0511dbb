// frontend_points.cu -- the tracked frame's bookkeeping on sm_90a: matchAndTrack's candidate groups and budget
// (scavislam/stereo_frontend.cpp:977-1065), processMatchedPoints (:834-974), shallWeDropNewKeyframe (:512-528) and the
// point seeding of addMorePointsToOtherFrame (:724-823).
//
// Kernels: the budget's stop rule and processMatchedPoints are one small CTA each (sequential over the groups / in
// match order, so counts, order and the double track-length sum are exact).  The seeding runs one CTA per matcher level
// over that level's FAST corners in global scratch: the full-depth quadtree path of every corner; its position in
// (path, index) order by counting; per depth, the first thread of every node (a run of equal path prefixes) picks the
// node's emission; the emission order by counting; then the reference's sequential greedy (a corner is taken when no
// tree point and no earlier taken corner lies in its window) as rounds of an exact fixed point over a bucket grid; the
// per-level cap in one pass.  The two counting ranks are O(n^2 / threads) for n corners of a level.  The projections are compiled with
// -fmad=false and written operation by operation like oracle/frontend_oracle.c.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/svs_b200.h"
#include "internal.cuh"
#include "se3_dev.cuh"
#include "svs_nvtx.hpp"

namespace {

constexpr int kLv = SVS_MATCH_MAX_LEVELS;
constexpr int kCta = 256;       // the budget and process CTAs
constexpr int kSeed = 512;      // the seeding CTA of one level
constexpr int kDepth = 16;      // quadtree depth at which distinct integer positions of a level < 65536 px separate

struct Pose7 { double v[7]; };

struct ProcArgs {
  Pose7 T;
  double f, px, py, b;
  int w0, h0, n, n_new;
  float max_err;
  int min_num_points;
};

// the device image of svs_point_stats and the add flags (written by k_process)
struct ProcOut {
  svs_point_stats st;
  int flags[9];
};

struct SeedArgs {
  int w0, h0;                    // level 0
  int wl[kLv], hl[kLv], nkp[kLv], cap[kLv], out_off[kLv];
  const int* kp_xy[kLv];
  const float* disp;
  int disp_pitch;
  int R, fresh, slot;
  unsigned long long seed;
  const ProcOut* proc;           // fresh = 0: flags and num_matched_points
  const svs_tracked_point* trk;  // fresh = 0: the gated points (the tree)
  const int* n_trk;              // fresh = 0: their count (device)
  Pose7 T;
  double f, px, py, b;
};

// per-level scratch of the seeding (level l at offset l * stride of each array)
struct SeedScratch {
  unsigned long long *key, *nh;  // [max_kp] corner key, node hash at the emission depth
  unsigned* path;                // [max_kp] full-depth path
  int *spos, *edepth, *order, *rank, *status, *outk;   // [max_kp]
  int* cell_ptr;                 // [ncell_max + 1]
  int* cell_cur;                 // [ncell_max]
  int* cell_item;                // [max_kp + max_pts]
  size_t stride_kp, stride_cell, stride_item;
};

__device__ __forceinline__ unsigned long long sm64(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ull;
  unsigned long long z = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ unsigned long long hash5(unsigned long long a, unsigned long long b, unsigned long long c,
                                                    unsigned long long d, unsigned long long e) {
  return sm64(sm64(sm64(sm64(sm64(a) ^ b) ^ c) ^ d) ^ e);
}

// cv::Rect_<double>(cx - R, cy - R, 2R+1, 2R+1).contains(p)
__device__ __forceinline__ bool in_win(double cx, double cy, int R, double px, double py) {
  const double x0 = cx - R, y0 = cy - R, d = 2 * R + 1;
  return x0 <= px && px < x0 + d && y0 <= py && py < y0 + d;
}

// ------------------------------------------------------------------ matchAndTrack's stop rule
// One CTA walks the groups in order: group g's matched count is a block reduction; a neighbour group that is not kept
// has its entries' matched cleared.  cnt[0] = num_new_feat_matched, cnt[1] = num_obs.
__global__ void __launch_bounds__(kCta) k_budget(svs_match_result* __restrict__ res, int n_groups,
                                                 const int* __restrict__ group_end, int num_max_points, int* __restrict__ cnt) {
  __shared__ int s_sum[kCta / 32];
  int total = 0, keep = 1, num_new = 0;
  for (int g = 0; g < n_groups; ++g) {
    const int b0 = g == 0 ? 0 : group_end[g - 1], b1 = group_end[g];
    const bool neighbour = g > 0 && g < n_groups - 1;
    if (neighbour) keep = keep && 2 * total < num_max_points;
    int c = 0;
    for (int i = b0 + threadIdx.x; i < b1; i += kCta) {
      if (neighbour && !keep) res[i].matched = 0;
      c += res[i].matched;
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = c;
    __syncthreads();
    int s = 0;
    for (int k = 0; k < kCta / 32; ++k) s += s_sum[k];
    __syncthreads();
    total += s;
    if (g == n_groups - 2) num_new = total;
  }
  if (threadIdx.x == 0) { cnt[0] = num_new; cnt[1] = total; }
}

// ------------------------------------------------------------------ processMatchedPoints
__global__ void __launch_bounds__(kCta) k_process(const svs_match_result* __restrict__ res, const svs_match_point* __restrict__ pts,
                                                  ProcArgs a, svs_tracked_point* __restrict__ trk, double* __restrict__ term,
                                                  int* __restrict__ n_trk, ProcOut* __restrict__ out) {
  __shared__ int sw[kCta / 32];
  __shared__ int carry;
  __shared__ int g2[4], g3[9], nm[kLv], nnew;
  if (threadIdx.x < 4) g2[threadIdx.x] = 0;
  if (threadIdx.x < 9) g3[threadIdx.x] = 0;
  if (threadIdx.x < kLv) nm[threadIdx.x] = 0;
  if (threadIdx.x == 0) { carry = 0; nnew = 0; }
  double R[9];
  svs::quat_to_R(a.T.v, R);
  const int half_w = (int)(a.w0 * 0.5), half_h = (int)(a.h0 * 0.5);
  const float third = (float)(1. / 3.);
  const int tw = (int)((float)a.w0 * third), th = (int)((float)a.h0 * third);
  const int ttw = (int)((float)(a.w0 * 2) * third), tth = (int)((float)(a.h0 * 2) * third);
  __syncthreads();
  for (int base = 0; base < a.n; base += kCta) {
    const int i = base + threadIdx.x;
    int keep = 0, lvl = 0;
    double t = 0;
    if (i < a.n && res[i].matched) {
      const svs_match_result r = res[i];
      lvl = pts[i].anchor_level;
      const int factor = 1 << lvl;
      const double thr_uv = (double)(a.max_err * (float)factor);
      const double thr_r = 3. * (double)a.max_err;
      if (svs::reproj_gate(r, R, a.T.v, a.f, a.px, a.py, a.b, thr_uv, thr_r)) {
        keep = 1;
        const int i2 = r.obs[0] < half_w ? 0 : 1, j2 = r.obs[1] < half_h ? 0 : 1;
        atomicAdd(&g2[i2 * 2 + j2], 1);
        const int i3 = r.obs[0] < tw ? 0 : (r.obs[0] < ttw ? 1 : 2);
        const int j3 = r.obs[1] < th ? 0 : (r.obs[1] < tth ? 1 : 2);
        atomicAdd(&g3[i3 * 3 + j3], 1);
        atomicAdd(&nm[lvl], 1);
        if (i < a.n_new) atomicAdd(&nnew, 1);
        // curkey_uv_pyr = SE3XYZ::map(SE3(), xyz) / 2^level, uv_pyr = uvu.xy / 2^level
        const double s = (double)factor;
        const double X0 = r.xyz_actkey[0], X1 = r.xyz_actkey[1], X2 = r.xyz_actkey[2];
        const double cu = (a.f * (X0 / X2) + a.px) / s, cv = (a.f * (X1 / X2) + a.py) / s;
        const double du = r.obs[0] / s - cu, dv = r.obs[1] / s - cv;
        t = sqrt(du * du + dv * dv);
      }
    }
    int sc = keep;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, sc, o); if ((threadIdx.x & 31) >= o) sc += v; }
    if ((threadIdx.x & 31) == 31) sw[threadIdx.x >> 5] = sc;
    __syncthreads();
    int before = 0;
    for (int k = 0; k < (int)(threadIdx.x >> 5); ++k) before += sw[k];
    const int at = carry + before + sc - keep;
    if (keep) {
      svs_tracked_point p;
      p.index = i; p.is_new = i < a.n_new; p.anchor_level = lvl; p.reserved = 0;
      p.uvu[0] = res[i].obs[0]; p.uvu[1] = res[i].obs[1]; p.uvu[2] = res[i].obs[2];
      trk[at] = p;
      term[at] = t;
    }
    __syncthreads();
    if (threadIdx.x == kCta - 1) carry = at + keep;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    // the reference's sum runs in match order in double: sequential here
    double sum = 0.;
    for (int k = 0; k < carry; ++k) sum += term[k];
    svs_point_stats st;
    memset(&st, 0, sizeof st);
    for (int l = 0; l < kLv; ++l) st.num_matched_points[l] = nm[l];
    for (int k = 0; k < 4; ++k) st.grid2x2[k >> 1][k & 1] = g2[k];
    for (int k = 0; k < 9; ++k) st.grid3x3[k / 3][k % 3] = g3[k];
    st.av_track_length = sum / (double)carry;
    st.num_tracked = carry;
    st.num_new = nnew;
    out->st = st;
    for (int k = 0; k < 9; ++k) out->flags[k] = g3[k] <= a.min_num_points;
    *n_trk = carry;
  }
}

// the per-handle state: the gated points of the last processMatchedPoints (valid for the match it followed)
// one CTA per level: the seeding of addMorePointsToOtherFrame (see svs_addMorePoints)
__global__ void __launch_bounds__(kSeed, 1) k_seed(const __grid_constant__ SeedArgs a, const __grid_constant__ SeedScratch sc,
                                                   svs_new_point* __restrict__ out_pts, svs_match_point* __restrict__ out_rows,
                                                   int* __restrict__ counts) {
  const int l = blockIdx.x, tid = threadIdx.x;
  const int n = a.nkp[l];
  const int* __restrict__ xy = a.kp_xy[l];
  unsigned long long* key = sc.key + l * sc.stride_kp;
  unsigned long long* nh = sc.nh + l * sc.stride_kp;
  unsigned* path = sc.path + l * sc.stride_kp;
  int* spos = sc.spos + l * sc.stride_kp;
  int* ed = sc.edepth + l * sc.stride_kp;
  int* order = sc.order + l * sc.stride_kp;
  int* rank = sc.rank + l * sc.stride_kp;
  int* status = sc.status + l * sc.stride_kp;   // 0 undecided, 1 taken, 2 refused, 3 not a candidate, 4 emitted
  int* outk = sc.outk + l * sc.stride_kp;
  int* cell_ptr = sc.cell_ptr + l * sc.stride_cell;
  int* cell_cur = sc.cell_cur + l * sc.stride_cell;
  int* cell_item = sc.cell_item + l * sc.stride_item;
  __shared__ int s_m;
  // ---- corner keys and full-depth paths
  for (int i = tid; i < n; i += kSeed) {
    const int u = xy[2 * i], v = xy[2 * i + 1];
    key[i] = hash5(a.seed, 0ull, (unsigned long long)l, (unsigned long long)u, (unsigned long long)v);
    double x = 0, y = 0, w = a.wl[l], h = a.hl[l];
    unsigned P = 0;
    for (int d = 0; d < kDepth; ++d) {
      const double x1 = x + w * 0.5, y1 = y + h * 0.5;
      const unsigned bx = u >= x1, by = v >= y1;
      if (bx) x = x1;
      if (by) y = y1;
      w = w * 0.5; h = h * 0.5;
      P = (P << 2) | (bx << 1) | by;
    }
    path[i] = P;
    ed[i] = INT_MAX;
  }
  __syncthreads();
  // ---- position in (path, index) order: the nodes of every depth are runs of it
  for (int i = tid; i < n; i += kSeed) {
    const unsigned P = path[i];
    int pos = 0;
    for (int j = 0; j < n; ++j) {
      const unsigned Q = path[j];
      pos += Q < P || (Q == P && j < i);
    }
    spos[pos] = i;
  }
  __syncthreads();
  // of corners at one position (one full-depth node) only the lowest index exists
  for (int p = tid; p < n; p += kSeed) status[spos[p]] = p > 0 && path[spos[p - 1]] == path[spos[p]] ? 3 : 0;
  __syncthreads();
  // ---- emission depths: the first thread of every node at depth d emits the node's smallest (key, index)
  for (int d = 0; d <= kDepth; ++d) {
    const int sh = 2 * (kDepth - d);
    for (int p = tid; p < n; p += kSeed) {
      const unsigned long long pre = (unsigned long long)path[spos[p]] >> sh;
      if (p > 0 && ((unsigned long long)path[spos[p - 1]] >> sh) == pre) continue;
      int best = -1;
      for (int q = p; q < n && ((unsigned long long)path[spos[q]] >> sh) == pre; ++q) {
        const int c = spos[q];
        if (status[c] != 0) continue;
        if (best < 0 || key[c] < key[best] || (key[c] == key[best] && c < best)) best = c;
      }
      if (best >= 0) {
        status[best] = 4;
        ed[best] = d;
        nh[best] = hash5(a.seed, 1ull, (unsigned long long)l, (unsigned long long)d, pre);
      }
    }
    __syncthreads();
  }
  // ---- emission order: (depth, node hash, path prefix) by counting over the emitted corners
  if (tid == 0) s_m = 0;
  __syncthreads();
  for (int c = tid; c < n; c += kSeed) {
    if (status[c] != 4) continue;
    atomicAdd(&s_m, 1);
    const int dc = ed[c];
    const unsigned long long hc = nh[c], pc = (unsigned long long)path[c] >> (2 * (kDepth - dc));
    int r = 0;
    for (int j = 0; j < n; ++j) {
      if (status[j] != 4 || j == c) continue;
      const int dj = ed[j];
      if (dj != dc) { r += dj < dc; continue; }
      const unsigned long long hj = nh[j];
      if (hj != hc) { r += hj < hc; continue; }
      r += ((unsigned long long)path[j] >> (2 * (kDepth - dj))) < pc;
    }
    order[r] = c;
    rank[c] = r;
  }
  __syncthreads();
  const int m = s_m;
  // ---- the filters of addMorePointsToOtherFrame (order-free)
  const float third = (float)(1. / 3.);
  const int tw = (int)((float)a.w0 * third), th = (int)((float)a.h0 * third);
  const int ttw = (int)((float)(a.w0 * 2) * third), tth = (int)((float)(a.h0 * 2) * third);
  const double inv_factor = 1. / (double)(1 << l), sl = (double)(1 << l);
  for (int c = tid; c < n; c += kSeed) {
    outk[c] = -1;
    if (status[c] != 4) { status[c] = 3; continue; }
    const int uz = xy[2 * c] << l, vz = xy[2 * c + 1] << l;
    const double disp = uz < a.w0 && vz < a.h0 ? (double)a.disp[(size_t)vz * a.disp_pitch + uz] * inv_factor : 0.;
    bool ok = disp > 0 && uz >= 1 && uz < a.w0 - 1 && vz >= 1 && vz < a.h0 - 1;
    if (ok) {
      const int i3 = uz < tw ? 0 : (uz < ttw ? 1 : 2), j3 = vz < th ? 0 : (vz < tth ? 1 : 2);
      ok = a.fresh || a.proc->flags[i3 * 3 + j3];
    }
    status[c] = ok ? 0 : 3;
  }
  // ---- bucket grid of the candidates and the level's tree points; cell >= 2R+1 so a window spans <= 2 cells per axis
  const int cs = max(2 * a.R + 1, 8);
  const int gw = a.wl[l] / cs + 1, gh = a.hl[l] / cs + 1, ncell = gw * gh;
  const int ntrk = a.fresh ? 0 : *a.n_trk;
  for (int k = tid; k < ncell; k += kSeed) cell_cur[k] = 0;
  __syncthreads();
  auto cell_of = [=](double x, double y) {
    const int cx = min(max((int)floor(x / cs), 0), gw - 1), cy = min(max((int)floor(y / cs), 0), gh - 1);
    return cy * gw + cx;
  };
  for (int i = tid; i < n + ntrk; i += kSeed) {
    if (i < n) {
      if (status[i] == 0) atomicAdd(&cell_cur[cell_of(xy[2 * i], xy[2 * i + 1])], 1);
    } else if (a.trk[i - n].anchor_level == l) {
      atomicAdd(&cell_cur[cell_of(a.trk[i - n].uvu[0] / sl, a.trk[i - n].uvu[1] / sl)], 1);
    }
  }
  __syncthreads();
  if (tid == 0) {
    int run = 0;
    for (int k = 0; k < ncell; ++k) { cell_ptr[k] = run; run += cell_cur[k]; cell_cur[k] = cell_ptr[k]; }
    cell_ptr[ncell] = run;
  }
  __syncthreads();
  for (int i = tid; i < n + ntrk; i += kSeed) {
    if (i < n) {
      if (status[i] == 0) cell_item[atomicAdd(&cell_cur[cell_of(xy[2 * i], xy[2 * i + 1])], 1)] = i;
    } else if (a.trk[i - n].anchor_level == l) {
      cell_item[atomicAdd(&cell_cur[cell_of(a.trk[i - n].uvu[0] / sl, a.trk[i - n].uvu[1] / sl)], 1)] = i;
    }
  }
  __syncthreads();
  // ---- the greedy in emission order as rounds: a candidate is refused once a lower-rank candidate in its window is
  // taken (or a tree point lies there) and taken once every lower-rank candidate in its window is refused.  Statuses
  // only move from undecided to final, so reading another thread's fresh write is as good as the next round's read;
  // the lowest-rank undecided candidate always decides, so the rounds end.
  volatile int* st = status;
  for (;;) {
    int left = 0;
    for (int c = tid; c < n; c += kSeed) {
      if (st[c] != 0) continue;
      const double cx = xy[2 * c], cy = xy[2 * c + 1];
      const int x0 = min(max((int)floor((cx - a.R) / cs), 0), gw - 1), x1 = min(max((int)floor((cx + a.R + 1) / cs), 0), gw - 1);
      const int y0 = min(max((int)floor((cy - a.R) / cs), 0), gh - 1), y1 = min(max((int)floor((cy + a.R + 1) / cs), 0), gh - 1);
      int verdict = 1;
      for (int gy = y0; gy <= y1 && verdict != 2; ++gy)
        for (int gx = x0; gx <= x1 && verdict != 2; ++gx) {
          const int cell = gy * gw + gx;
          for (int e = cell_ptr[cell]; e < cell_ptr[cell + 1]; ++e) {
            const int j = cell_item[e];
            if (j >= n) {
              if (in_win(cx, cy, a.R, a.trk[j - n].uvu[0] / sl, a.trk[j - n].uvu[1] / sl)) { verdict = 2; break; }
              continue;
            }
            if (j == c || rank[j] > rank[c] || !in_win(cx, cy, a.R, xy[2 * j], xy[2 * j + 1])) continue;
            const int sj = st[j];
            if (sj == 1) { verdict = 2; break; }
            if (sj == 0) verdict = 0;
          }
        }
      if (verdict) st[c] = verdict; else left = 1;
    }
    if (!__syncthreads_or(left)) break;
  }
  // ---- the cap: taken candidates in emission order until one makes the count exceed cap
  if (tid == 0) {
    const int n_in = a.fresh ? 0 : a.proc->st.num_matched_points[l];
    const int limit = max(1, a.cap[l] + 1 - n_in);
    int k = 0;
    for (int r = 0; r < m && k < limit; ++r)
      if (status[order[r]] == 1) outk[order[r]] = k++;
    counts[l] = k;
  }
  __syncthreads();
  for (int c = tid; c < n; c += kSeed) {
    const int k = outk[c];
    if (k < 0) continue;
    const double u = xy[2 * c], v = xy[2 * c + 1];
    const double disp = (double)a.disp[(size_t)(xy[2 * c + 1] << l) * a.disp_pitch + (xy[2 * c] << l)] * inv_factor;
    const double up = u - disp;
    // zeroFromPyr_3d, StereoCamera::unmap_uvu (stereo_camera.cpp:46-52)
    const double u0 = u * sl, v0 = v * sl, r0 = up * sl;
    const double sd = (u0 - r0) / a.b;
    const double z = a.f / sd;
    double xc[3], xw[3], Rm[9];
    xc[0] = (u0 - a.px) / a.f * z;
    xc[1] = (v0 - a.py) / a.f * z;
    xc[2] = z;
    svs::quat_to_R(a.T.v, Rm);
    svs::mat3_vec(Rm, xc, xw);
    xw[0] += a.T.v[4]; xw[1] += a.T.v[5]; xw[2] += a.T.v[6];
    const double dist = sqrt(xc[0] * xc[0] + xc[1] * xc[1] + xc[2] * xc[2]);
    svs_new_point* p = out_pts + a.out_off[l] + k;
    p->level = l; p->reserved = 0;
    p->uv_pyr[0] = u; p->uv_pyr[1] = v;
    p->uvu_pyr[0] = u; p->uvu_pyr[1] = v; p->uvu_pyr[2] = up;
    for (int q = 0; q < 3; ++q) { p->xyz[q] = xw[q]; p->normal[q] = -xc[q] / dist; }
    svs_match_point* mp = out_rows + a.out_off[l] + k;
    mp->keyframe = a.slot; mp->anchor_level = l;
    for (int q = 0; q < 3; ++q) mp->xyz_anchor[q] = xw[q];
    mp->anchor_obs_pyr[0] = u; mp->anchor_obs_pyr[1] = v;
  }
}

}  // namespace

struct svs::FrontState {
  unsigned long long serial = 0;   // match_serial the processed points belong to; 0: none
  svs_tracked_point* d_trk = nullptr;
  double* d_term = nullptr;
  int* d_cnt = nullptr;            // [0] gated count, [1..2] budget counts
  ProcOut* d_proc = nullptr;
  int* d_group_end = nullptr;
  size_t group_cap = 0;
  // seeding
  void* d_scratch = nullptr;
  SeedScratch sc{};
  svs_new_point* d_out_pts = nullptr;
  svs_match_point* d_out_rows = nullptr;
  int* d_counts = nullptr;
  size_t pts_cap = 0, rows_cap = 0;
};

void svs::front_state_free(FrontState* s) {
  if (!s) return;
  cudaFree(s->d_trk); cudaFree(s->d_term); cudaFree(s->d_cnt); cudaFree(s->d_proc); cudaFree(s->d_group_end);
  cudaFree(s->d_scratch); cudaFree(s->d_out_pts); cudaFree(s->d_out_rows); cudaFree(s->d_counts);
  delete s;
}

// the state with the buffers every call needs (allocated once per handle)
static int front_state(const svs::MatcherCore& c, svs::FrontState** out) {
  if (!*c.front) {
    // published only once every buffer is there: a failed allocation leaves no half-made state behind
    svs::FrontState* s = new svs::FrontState();
    const bool ok = cudaMalloc(&s->d_trk, sizeof(svs_tracked_point) * (size_t)c.max_pts) == cudaSuccess &&
                    cudaMalloc(&s->d_term, sizeof(double) * (size_t)c.max_pts) == cudaSuccess &&
                    cudaMalloc(&s->d_cnt, sizeof(int) * 4) == cudaSuccess &&
                    cudaMalloc(&s->d_proc, sizeof(ProcOut)) == cudaSuccess;
    if (!ok) {
      svs::front_state_free(s);
      cudaGetLastError();
      return svs::fail(c.base, SVS_ERR_CUDA, "frontend: out of device memory for the state buffers");
    }
    *c.front = s;
  }
  *out = *c.front;
  return SVS_OK;
}

static bool pose_ok(const double* T) {
  if (!T) return false;
  for (int k = 0; k < 7; ++k)
    if (!std::isfinite(T[k])) return false;
  return true;
}

static bool params_ok(const svs_frontend_params* p) {
  return p && p->newpoint_clearance >= 0 && p->newpoint_clearance <= 64 && p->num_max_points >= 0 &&
         std::isfinite(p->max_reproj_error) && p->max_reproj_error >= 0.f;
}

extern "C" {

int svs_match_track(svs_matcher* m, const double T_cur_from_actkey[7], const double T_actkey_from_w[7],
                    const svs_match_point* pts, int n, int n_groups, const int* group_end, int num_max_points,
                    int search_radius, int thr_mean, int thr_std, svs_match_result* out, int* num_new_feat_matched,
                    int* num_obs) {
  svs::NvtxRange nvtx_("match_track");
  if (!m) return SVS_ERR_INVALID;
  svs::MatcherCore c;
  svs::matcher_core(m, &c);
  if (!T_cur_from_actkey || !T_actkey_from_w || n < 0 || n > c.max_pts || (n && !pts) || search_radius < 0 ||
      n_groups < 2 || !group_end)
    return svs::fail(c.base, SVS_ERR_INVALID, "match_track: bad pose, point count, radius or groups");
  for (int g = 0; g < n_groups; ++g)
    if (group_end[g] < (g ? group_end[g - 1] : 0) || group_end[g] > n)
      return svs::fail(c.base, SVS_ERR_INVALID, "match_track: group_end must be non-decreasing within [0, n]");
  if (group_end[n_groups - 1] != n) return svs::fail(c.base, SVS_ERR_INVALID, "match_track: group_end[n_groups-1] != n");
  cudaSetDevice(c.device);
  svs::FrontState* s;
  int rc = front_state(c, &s);
  if (rc != SVS_OK) return rc;
  SVS_CK(c.base, svs::grow((size_t)n_groups, &s->group_cap, &s->d_group_end));
  if (n) SVS_CK(c.base, cudaMemcpyAsync(c.d_pts, pts, sizeof(svs_match_point) * (size_t)n, cudaMemcpyHostToDevice, c.stream));
  SVS_CK(c.base, cudaMemcpyAsync(s->d_group_end, group_end, sizeof(int) * (size_t)n_groups, cudaMemcpyHostToDevice, c.stream));
  rc = svs::match_enqueue_own(m, T_cur_from_actkey, T_actkey_from_w, n, search_radius, thr_mean, thr_std);
  if (rc != SVS_OK) return rc;
  k_budget<<<1, kCta, 0, c.stream>>>(c.d_res, n_groups, s->d_group_end, num_max_points, s->d_cnt + 1);
  SVS_CK(c.base, cudaGetLastError());
  int cnt[2];
  SVS_CK(c.base, cudaMemcpyAsync(cnt, s->d_cnt + 1, sizeof cnt, cudaMemcpyDeviceToHost, c.stream));
  if (out && n) SVS_CK(c.base, cudaMemcpyAsync(out, c.d_res, sizeof(svs_match_result) * (size_t)n, cudaMemcpyDeviceToHost, c.stream));
  SVS_CK(c.base, cudaStreamSynchronize(c.stream));
  if (num_new_feat_matched) *num_new_feat_matched = cnt[0];
  if (num_obs) *num_obs = cnt[1];
  return SVS_OK;
}

int svs_shallWeDropNewKeyframe(const svs_point_stats* st, const double T[7], const svs_frontend_params* p) {
  if (!st || !T || !p) return SVS_ERR_INVALID;
  int featureless = 0;
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j)
      if (st->grid2x2[i][j] < 15) ++featureless;
  const double tn = std::sqrt(T[4] * T[4] + T[5] * T[5] + T[6] * T[6]);
  return featureless > p->featureless_corners_thr || tn > p->parallax_thr || st->av_track_length > 75.;
}

int svs_processMatchedPoints(svs_matcher* m, const double T_cur_from_actkey[7], const svs_cam* cam, int n_new,
                             const svs_frontend_params* params, svs_tracked_point* out, svs_point_stats* stats,
                             int add_flags[9], int* drop_keyframe) {
  svs::NvtxRange nvtx_("process_points");
  if (!m) return SVS_ERR_INVALID;
  svs::MatcherCore c;
  svs::matcher_core(m, &c);
  if (!pose_ok(T_cur_from_actkey) || !cam || !params_ok(params) || n_new < 0)
    return svs::fail(c.base, SVS_ERR_INVALID, "processMatchedPoints: bad pose, camera, parameters or n_new");
  if (!c.match_serial || !c.last_pts_own)
    return svs::fail(c.base, SVS_ERR_STATE, "processMatchedPoints: needs a preceding svs_match or svs_match_track on this handle");
  if (n_new > c.last_n) return svs::fail(c.base, SVS_ERR_INVALID, "processMatchedPoints: n_new exceeds the candidates of the last match");
  cudaSetDevice(c.device);
  svs::FrontState* s;
  int rc = front_state(c, &s);
  if (rc != SVS_OK) return rc;
  s->serial = 0;
  ProcArgs a;
  memcpy(a.T.v, T_cur_from_actkey, sizeof(double) * 7);
  a.f = cam->f; a.px = cam->px; a.py = cam->py; a.b = cam->b;
  a.w0 = c.lv[0].w; a.h0 = c.lv[0].h; a.n = c.last_n; a.n_new = n_new;
  a.max_err = params->max_reproj_error; a.min_num_points = params->min_num_points;
  k_process<<<1, kCta, 0, c.stream>>>(c.d_res, c.d_pts, a, s->d_trk, s->d_term, s->d_cnt, s->d_proc);
  SVS_CK(c.base, cudaGetLastError());
  ProcOut po;
  SVS_CK(c.base, cudaMemcpyAsync(&po, s->d_proc, sizeof po, cudaMemcpyDeviceToHost, c.stream));
  SVS_CK(c.base, cudaStreamSynchronize(c.stream));
  const int ng = po.st.num_tracked;
  if (out && ng) {
    SVS_CK(c.base, cudaMemcpyAsync(out, s->d_trk, sizeof(svs_tracked_point) * (size_t)ng, cudaMemcpyDeviceToHost, c.stream));
    SVS_CK(c.base, cudaStreamSynchronize(c.stream));
  }
  s->serial = c.match_serial;
  if (stats) *stats = po.st;
  if (add_flags) memcpy(add_flags, po.flags, sizeof po.flags);
  if (drop_keyframe) *drop_keyframe = svs_shallWeDropNewKeyframe(&po.st, T_cur_from_actkey, params);
  return ng;
}

int svs_addMorePoints(svs_matcher* m, int fresh, const double T_newkey_from_cur[7], const svs_cam* cam, int keyframe_slot,
                      const svs_frontend_params* params, svs_new_point* points, svs_match_point* rows, int cap,
                      int* counts) {
  svs::NvtxRange nvtx_("add_more_points");
  if (!m) return SVS_ERR_INVALID;
  svs::MatcherCore c;
  svs::matcher_core(m, &c);
  if ((fresh != 0 && fresh != 1) || !pose_ok(T_newkey_from_cur) || !cam || !params_ok(params))
    return svs::fail(c.base, SVS_ERR_INVALID, "addMorePoints: bad mode, pose, camera or parameters");
  int bound = 0, off[kLv] = {};
  for (int l = 0; l < c.nlevels; ++l) { off[l] = bound; bound += (params->num_max_points >> l) + 1; }
  if ((points || rows) && cap < bound)
    return svs::fail(c.base, SVS_ERR_INVALID, "addMorePoints: cap below the sum over levels of (num_max_points >> l) + 1");
  for (int l = 0; l < c.nlevels; ++l)
    if (c.lv[l].w > 65535 || c.lv[l].h > 65535) return svs::fail(c.base, SVS_ERR_UNSUPPORTED, "addMorePoints: level wider than 65535");
  const svs::FrontState* s0 = *c.front;
  if (!fresh && (!s0 || !s0->serial || s0->serial != c.match_serial))
    return svs::fail(c.base, SVS_ERR_STATE, "addMorePoints: no svs_processMatchedPoints since the last match");
  cudaSetDevice(c.device);
  svs::FrontState* s;
  int rc = front_state(c, &s);
  if (rc != SVS_OK) return rc;
  if (!s->d_scratch) {
    int ncell = 0;
    for (int l = 0; l < c.nlevels; ++l) ncell = std::max(ncell, (c.lv[l].w / 8 + 1) * (c.lv[l].h / 8 + 1));
    SeedScratch& q = s->sc;
    q.stride_kp = (size_t)c.max_kp;
    q.stride_cell = (size_t)ncell + 1;
    q.stride_item = (size_t)c.max_kp + c.max_pts;
    const size_t L = (size_t)c.nlevels;
    auto carve = [&](svs::Bump m) {
      q.key = m.take<unsigned long long>(L * q.stride_kp); q.nh = m.take<unsigned long long>(L * q.stride_kp);
      q.path = m.take<unsigned>(L * q.stride_kp);
      q.spos = m.take<int>(L * q.stride_kp); q.edepth = m.take<int>(L * q.stride_kp); q.order = m.take<int>(L * q.stride_kp);
      q.rank = m.take<int>(L * q.stride_kp); q.status = m.take<int>(L * q.stride_kp); q.outk = m.take<int>(L * q.stride_kp);
      q.cell_ptr = m.take<int>(L * q.stride_cell); q.cell_cur = m.take<int>(L * q.stride_cell);
      q.cell_item = m.take<int>(L * q.stride_item);
      return m.off;
    };
    SVS_CK(c.base, cudaMalloc(&s->d_scratch, carve(svs::Bump{nullptr})));
    carve(svs::Bump{static_cast<char*>(s->d_scratch)});
  }
  SVS_CK(c.base, svs::grow((size_t)bound, &s->pts_cap, &s->d_out_pts));
  SVS_CK(c.base, svs::grow((size_t)bound, &s->rows_cap, &s->d_out_rows));
  if (!s->d_counts) SVS_CK(c.base, cudaMalloc(&s->d_counts, sizeof(int) * kLv));
  SeedArgs a;
  memset(&a, 0, sizeof a);
  a.w0 = c.lv[0].w; a.h0 = c.lv[0].h;
  for (int l = 0; l < c.nlevels; ++l) {
    a.wl[l] = c.lv[l].w; a.hl[l] = c.lv[l].h; a.nkp[l] = c.nkp[l]; a.kp_xy[l] = c.d_kp_xy[l];
    a.cap[l] = params->num_max_points >> l; a.out_off[l] = off[l];
  }
  a.disp = c.d_disp; a.disp_pitch = c.disp_pitch;
  a.R = params->newpoint_clearance; a.seed = params->seed; a.fresh = fresh; a.slot = keyframe_slot;
  a.proc = s->d_proc; a.trk = s->d_trk; a.n_trk = s->d_cnt;
  memcpy(a.T.v, T_newkey_from_cur, sizeof(double) * 7);
  a.f = cam->f; a.px = cam->px; a.py = cam->py; a.b = cam->b;
  k_seed<<<c.nlevels, kSeed, 0, c.stream>>>(a, s->sc, s->d_out_pts, s->d_out_rows, s->d_counts);
  SVS_CK(c.base, cudaGetLastError());
  int cnt[kLv] = {};
  std::vector<svs_new_point> hp((size_t)bound);
  std::vector<svs_match_point> hr((size_t)bound);
  SVS_CK(c.base, cudaMemcpyAsync(cnt, s->d_counts, sizeof(int) * c.nlevels, cudaMemcpyDeviceToHost, c.stream));
  if (points) SVS_CK(c.base, cudaMemcpyAsync(hp.data(), s->d_out_pts, sizeof(svs_new_point) * (size_t)bound, cudaMemcpyDeviceToHost, c.stream));
  if (rows) SVS_CK(c.base, cudaMemcpyAsync(hr.data(), s->d_out_rows, sizeof(svs_match_point) * (size_t)bound, cudaMemcpyDeviceToHost, c.stream));
  SVS_CK(c.base, cudaStreamSynchronize(c.stream));
  int total = 0;
  for (int l = 0; l < c.nlevels; ++l) {
    if (points) memcpy(points + total, hp.data() + off[l], sizeof(svs_new_point) * (size_t)cnt[l]);
    if (rows) memcpy(rows + total, hr.data() + off[l], sizeof(svs_match_point) * (size_t)cnt[l]);
    total += cnt[l];
  }
  if (counts)
    for (int l = 0; l < kLv; ++l) counts[l] = l < c.nlevels ? cnt[l] : 0;
  return total;
}

}  // extern "C"
