// graph.cu -- the SLAM map kept on the device and the assembly of a double-window problem from it
// (SURVEY.md 8f rank 3, a "next" row): SlamGraph::copyDataToG2o / copyPosesToG2o / addPointToG2o /
// addObsToG2o (scavislam/slam_graph.cpp:907-1032, slam_graph-impl.cpp:29-126) without the O(E) walk over
// hash maps on the host: vertices (T_me_from_world), points (anchorframe_id, xyz_anchor) and the
// observations (vis_set + feature_table: centre and pyramid level) live in device memory; a window is
// assembled by three kernels (count the visible poses of every active point that lie in the window,
// exclusive scan, emit the edges in the reference's order: active points in list order, vis_set order inside)
// and handed to the bundle adjuster where it lies -- only the edge index triples come back to the host,
// for the structure analysis of svs_ba_set_problem.
//
// Round 2 adds what surrounds the assembly: the choice of the double window from the pose graph
// (computeInitialDoubleWin + computeActivePointsAndExtendOuterWindow, slam_graph.cpp:556-663, and the pair selection
// of copyContraintsToG2o, :938-981) and the growth of the map by one keyframe (addKeyframe, :144-186, 359-421), both
// on the tables where they lie.
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "../../include/svs_b200.h"
#include "handle.cuh"
#include "internal.cuh"
#include "se3_dev.cuh"
#include "svs_nvtx.hpp"

namespace {

struct MapDev {
  int V, Np;
  const double* pose;       // [V][7]
  const int* anchor;        // [Np] vertex index
  const double* xyz;        // [Np][3]
  const int* vis_ptr;       // [Np+1]
  const int* vis_pose;      // [nnz] vertex index
  const double* center;     // [nnz][3]  (u, v, u_right) at level 0
  const int* level;         // [nnz]
};

// edges of active point l = observations whose pose is in the window (slam_graph.cpp:1001-1027)
__global__ void k_count(MapDev m, const int* __restrict__ win_pos, const int* __restrict__ active, int L, int* __restrict__ cnt,
                        int* __restrict__ bad) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  const int p = active[l];
  if (win_pos[m.anchor[p]] < 0) atomicAdd(bad, 1);   // the anchor frame must be a vertex of the problem
  int c = 0;
  for (int i = m.vis_ptr[p]; i < m.vis_ptr[p + 1]; ++i) c += win_pos[m.vis_pose[i]] >= 0;
  cnt[l] = c;
}

// single-CTA exclusive scan (L is a few 10^4..10^5)
__global__ void k_scan(const int* __restrict__ cnt, int L, int* __restrict__ ptr) {
  __shared__ int sw[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < L; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const int v = i < L ? cnt[i] : 0;
    int s = v;
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, s, o); if ((threadIdx.x & 31) >= o) s += t; }
    if ((threadIdx.x & 31) == 31) sw[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
      int w = threadIdx.x < (blockDim.x >> 5) ? sw[threadIdx.x] : 0;
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, w, o); if (threadIdx.x >= o) w += t; }
      sw[threadIdx.x] = w;
    }
    __syncthreads();
    const int before = (threadIdx.x >> 5) ? sw[(threadIdx.x >> 5) - 1] : 0;
    if (i < L) ptr[i] = carry + before + s - v;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry += before + s;
    __syncthreads();
  }
  if (threadIdx.x == 0) ptr[L] = carry;
}

__global__ void k_emit(MapDev m, const int* __restrict__ win_pos, const int* __restrict__ active, int L,
                       const int* __restrict__ ptr, int E, int* __restrict__ e_point, int* __restrict__ e_pose,
                       int* __restrict__ e_anchor, double* __restrict__ obs_info, double* __restrict__ psi) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  const int p = active[l];
  {   // addPointToG2o: psi = invert_depth(xyz_anchor) (slam_graph.cpp:907-920, maths_utils.h:66-69)
    const double x = m.xyz[3 * (size_t)p], y = m.xyz[3 * (size_t)p + 1], z = m.xyz[3 * (size_t)p + 2];
    psi[3 * (size_t)l] = x / z; psi[3 * (size_t)l + 1] = y / z; psi[3 * (size_t)l + 2] = 1. / z;
  }
  const int a = win_pos[m.anchor[p]];
  int at = ptr[l];
  for (int i = m.vis_ptr[p]; i < m.vis_ptr[p + 1]; ++i) {
    const int w = win_pos[m.vis_pose[i]];
    if (w < 0) continue;
    e_point[at] = l; e_pose[at] = w; e_anchor[at] = a;
    double* o = obs_info + 3 * (size_t)at;
    o[0] = m.center[3 * (size_t)i]; o[1] = m.center[3 * (size_t)i + 1]; o[2] = m.center[3 * (size_t)i + 2];
    // Lambda = diag(s, s, 0.333^2), s = (2^-level)^2 (slam_graph.cpp:1010-1015)
    const double f = 1. / (double)(1 << m.level[i]), s = f * f;
    double* wq = obs_info + 3 * (size_t)E + 3 * (size_t)at;
    wq[0] = s; wq[1] = s; wq[2] = 0.333 * 0.333;
    ++at;
  }
}

__global__ void k_gather_poses(MapDev m, const int* __restrict__ window, int P, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 7 * P) return;
  out[i] = m.pose[7 * (size_t)window[i / 7] + i % 7];
}

// restoreDataFromG2o (slam_graph.cpp:1037-1058) without leaving the device: vertex and point estimates of the
// optimised window go back into the map (xyz_anchor = invert_depth(psi), maths_utils.h:66-69)
__global__ void k_absorb(double* __restrict__ map_pose, double* __restrict__ map_xyz, const double* __restrict__ pose0,
                         const double* __restrict__ pose1, const double* __restrict__ psi0, const double* __restrict__ psi1,
                         const int* __restrict__ lm_user, const int* __restrict__ cur, const int* __restrict__ window,
                         const int* __restrict__ active, int P, int L) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = *cur;
  const double* pose = c ? pose1 : pose0;
  const double* psi = c ? psi1 : psi0;
  if (i < 7 * P) map_pose[7 * (size_t)window[i / 7] + i % 7] = pose[i];
  if (i < L) {
    const double a = psi[3 * (size_t)i], b = psi[3 * (size_t)i + 1], w = psi[3 * (size_t)i + 2];
    double* x = map_xyz + 3 * (size_t)active[lm_user[i]];
    x[0] = a / w; x[1] = b / w; x[2] = 1. / w;
  }
}

// scatter of n records of `width` doubles into rows `index[i]` of a table
__global__ void k_scatter_rows(double* __restrict__ table, const int* __restrict__ index, const double* __restrict__ rows, int n,
                               int width) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * width) return;
  table[(size_t)width * index[i / width] + i % width] = rows[i];
}


// ------------------------------------------------------------------ window selection
struct GraphDev {
  const int* nbr_ptr;       // [V+1]
  const int* nbr_id;        // [nnzN] neighbours of a vertex, strongest first (the order computeInitialDoubleWin pushes them)
  const int* nbr_str;       // [nnzN] the strength key of neighbor_ids_ordered_by_strength (or nullptr)
  const double* nbr_T;      // [nnzN][7]  T_nbr_from_me of the directed entry (or nullptr)
  const double* nbr_Lam;    // [nnzN][36]
  const unsigned char* nbr_mrg;   // [nnzN] Edge::is_marginalized_ of the entry's edge (both entries carry it)
};

// computeInitialDoubleWin (slam_graph.cpp:556-598).  The queue discipline IS the algorithm (a vertex joins when it
// is popped, not when it is pushed), so one thread walks it; a window is a few hundred vertices.
__global__ void k_bfs(int V, GraphDev g, int root, int inner, int dbl, int* __restrict__ type, int* __restrict__ queue, int qcap) {
  if (blockIdx.x || threadIdx.x) return;
  int head = 0, tail = 0, count = 0;
  queue[tail++] = root;
  while (count < dbl && head < tail) {
    const int v = queue[head++];
    if (type[v]) continue;                       // "Avoid cycles!"
    type[v] = count < inner ? 1 : 2;
    ++count;
    for (int i = g.nbr_ptr[v]; i < g.nbr_ptr[v + 1] && tail < qcap; ++i) queue[tail++] = g.nbr_id[i];
  }
}

__device__ __forceinline__ bool has_edge(const GraphDev& g, int a, int b) {
  for (int i = g.nbr_ptr[a]; i < g.nbr_ptr[a + 1]; ++i)
    if (g.nbr_id[i] == b) return true;
  for (int i = g.nbr_ptr[b]; i < g.nbr_ptr[b + 1]; ++i)
    if (g.nbr_id[i] == a) return true;
  return false;
}

// computeActivePointsAndExtendOuterWindow (slam_graph.cpp:600-663), one thread per map point: active when an INNER
// frame sees it and its anchor frame is in the window, or that inner frame has an edge to the anchor frame (which then
// joins the outer window: ext[anchor] = 1)
__global__ void k_active(MapDev m, GraphDev g, const int* __restrict__ type, int* __restrict__ ext, int* __restrict__ active) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= m.Np) return;
  const int a = m.anchor[p];
  const bool inwin = type[a] != 0;
  int act = 0;
  for (int i = m.vis_ptr[p]; i < m.vis_ptr[p + 1] && !act; ++i) {
    const int f = m.vis_pose[i];
    if (type[f] != 1) continue;
    if (inwin) act = 1;
    else if (has_edge(g, f, a)) { act = 1; ext[a] = 1; }
  }
  active[p] = act;
}

__global__ void k_window_flags(int V, const int* __restrict__ type, const int* __restrict__ ext, int* __restrict__ wtype,
                               int* __restrict__ flag) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int t = type[v] ? type[v] : (ext[v] ? 2 : 0);
  wtype[v] = t;
  flag[v] = t != 0;
}

// out[ptr[i]] = i for flagged i (ascending: the order of a std::map / of the sorted point ids); pos[i] = ptr[i] or -1
__global__ void k_compact(int n, const int* __restrict__ flag, const int* __restrict__ ptr, int* __restrict__ out, int* __restrict__ pos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (flag[i]) out[ptr[i]] = i;
  if (pos) pos[i] = flag[i] ? ptr[i] : -1;
}

// the pair loop of copyContraintsToG2o (slam_graph.cpp:938-981) over the directed neighbour entries
__device__ __forceinline__ bool pair_selected(const int* wtype, int a, int b) {
  return b != a && wtype[a] && wtype[b] && (wtype[a] == 2 || wtype[b] == 2);
}
__global__ void k_pair_count(int V, GraphDev g, const int* __restrict__ wtype, int* __restrict__ cnt) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= V) return;
  int c = 0;
  for (int i = g.nbr_ptr[a]; i < g.nbr_ptr[a + 1]; ++i) c += pair_selected(wtype, a, g.nbr_id[i]);
  cnt[a] = c;
}
__global__ void k_pair_emit(int V, GraphDev g, const int* __restrict__ wtype, const int* __restrict__ win_pos,
                            const int* __restrict__ ptr, int* __restrict__ c_i, int* __restrict__ c_j, double* __restrict__ c_T,
                            double* __restrict__ c_Lam) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= V) return;
  for (int i = g.nbr_ptr[a]; i < g.nbr_ptr[a + 1]; ++i) {
    const int b = g.nbr_id[i];
    if (!pair_selected(wtype, a, b)) continue;
    int rank = 0;   // ascending id2 inside id1 (the inner loop of the reference runs over a std::map)
    for (int k = g.nbr_ptr[a]; k < g.nbr_ptr[a + 1]; ++k) rank += pair_selected(wtype, a, g.nbr_id[k]) && g.nbr_id[k] < b;
    const int at = ptr[a] + rank;
    c_i[at] = win_pos[a]; c_j[at] = win_pos[b];
    for (int q = 0; q < 7; ++q) c_T[7 * (size_t)at + q] = g.nbr_T ? g.nbr_T[7 * (size_t)i + q] : (q == 3 ? 1. : 0.);
    for (int q = 0; q < 36; ++q) c_Lam[36 * (size_t)at + q] = g.nbr_Lam ? g.nbr_Lam[36 * (size_t)i + q] : 0.;
  }
}

// ------------------------------------------------------------------ growth by one keyframe
// T_new = T_newkey_from_oldkey * T_oldkey_from_world (slam_graph.cpp:153-156)
__global__ void k_new_pose(const double* __restrict__ old_pose, int oldkey, const double* __restrict__ T_rel, double* __restrict__ out) {
  if (blockIdx.x || threadIdx.x) return;
  double A[7], B[7], AB[7];
  for (int q = 0; q < 7; ++q) { A[q] = T_rel[q]; B[q] = old_pose[7 * (size_t)oldkey + q]; }
  svs::se3_mul(A, B, AB);
  for (int q = 0; q < 7; ++q) out[q] = AB[q];
}
__device__ __forceinline__ bool observes(const MapDev& m, int p, int v) {
  for (int i = m.vis_ptr[p]; i < m.vis_ptr[p + 1]; ++i)
    if (m.vis_pose[i] == v) return true;
  return false;
}
// a tracked point gains an observation by `vertex` unless it has one already (std::map::insert keeps the old one)
__global__ void k_grow_count(MapDev m, int Np_new, int vertex, const int* __restrict__ add_idx, int* __restrict__ cnt) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Np_new) return;
  cnt[p] = p < m.Np ? m.vis_ptr[p + 1] - m.vis_ptr[p] + (add_idx[p] >= 0 && !observes(m, p, vertex)) : 2;
}
__global__ void k_mark_tracks(int n, const int* __restrict__ track_point, int* __restrict__ add_idx) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) add_idx[track_point[t]] = t;
}
// one thread per point moves its observations to their new place and inserts the tracked vertex's before the first
// observation by a larger vertex (a new keyframe's id is the largest: it goes last); a new point is seen by its anchor
// frame and the keyframe
__global__ void k_grow_move(MapDev m, int Np_new, int newkey, const int* __restrict__ add_idx, const int* __restrict__ new_ptr,
                            const double* __restrict__ track_center, const int* __restrict__ track_level,
                            const int* __restrict__ new_anchor, const double* __restrict__ new_anchor_center,
                            const int* __restrict__ new_anchor_level, const double* __restrict__ new_center,
                            const int* __restrict__ new_level, int* __restrict__ vis_pose, double* __restrict__ center,
                            int* __restrict__ level) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Np_new) return;
  int at = new_ptr[p];
  auto put = [&](int v, const double* c, int l) {
    vis_pose[at] = v; level[at] = l;
    center[3 * (size_t)at] = c[0]; center[3 * (size_t)at + 1] = c[1]; center[3 * (size_t)at + 2] = c[2];
    ++at;
  };
  if (p < m.Np) {
    const int t = add_idx[p];
    bool pending = t >= 0 && !observes(m, p, newkey);
    for (int i = m.vis_ptr[p]; i < m.vis_ptr[p + 1]; ++i) {
      if (pending && m.vis_pose[i] > newkey) { put(newkey, track_center + 3 * (size_t)t, track_level[t]); pending = false; }
      put(m.vis_pose[i], m.center + 3 * (size_t)i, m.level[i]);
    }
    if (pending) put(newkey, track_center + 3 * (size_t)t, track_level[t]);
  } else {
    const int q = p - m.Np;
    put(new_anchor[q], new_anchor_center + 3 * (size_t)q, new_anchor_level[q]);
    put(newkey, new_center + 3 * (size_t)q, new_level[q]);
  }
}

// ------------------------------------------------------------------ growth of the pose graph
// computeStrength (slam_graph.cpp:468-552), one record per (track, observer) pair: key (vertex, track), the quadrant
// bits of the track's centre (1 left / 2 right by u < half_width, 4 top / 8 bottom by v < half_height)
__global__ void k_str_count(MapDev m, int n_track, const int* __restrict__ track_point, int* __restrict__ cnt) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n_track) cnt[t] = m.vis_ptr[track_point[t] + 1] - m.vis_ptr[track_point[t]];
}
__global__ void k_str_emit(MapDev m, int n_track, const int* __restrict__ track_point, const double* __restrict__ track_center,
                           double half_w, double half_h, const int* __restrict__ ptr, unsigned long long* __restrict__ key,
                           unsigned char* __restrict__ quad, int* __restrict__ vcnt) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_track) return;
  const int p = track_point[t];
  const unsigned char q = (track_center[3 * (size_t)t] < half_w ? 1 : 2) | (track_center[3 * (size_t)t + 1] < half_h ? 4 : 8);
  int at = ptr[t];
  for (int i = m.vis_ptr[p]; i < m.vis_ptr[p + 1]; ++i, ++at) {
    const int v = m.vis_pose[i];
    key[at] = (unsigned long long)v << 32 | (unsigned)t;
    quad[at] = q;
    atomicAdd(vcnt + v, 1);
  }
}
__global__ void k_str_new(int n_new, const int* __restrict__ new_anchor, int* __restrict__ newcnt) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q < n_new) atomicAdd(newcnt + new_anchor[q], 1);
}
// Quirk B15 in closed form, one warp per vertex over its records in track order: the zeroing loop runs after every
// track, so a frame keeps only the tracks from t* on, t* = the first track after which its four quadrant counts are all
// >= need = max(1, covis_thr / 2); none: 0.  Without tracks the zeroing never runs and the new points stay.
__global__ void k_str_closed(int V, int n_track, int need, const int* __restrict__ vptr, const unsigned char* __restrict__ quad,
                             const int* __restrict__ newcnt, int* __restrict__ strength, int* __restrict__ in_table) {
  const int v = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (v >= V) return;
  const int s0 = vptr[v], s1 = vptr[v + 1];
  int tstar = -1, c0 = 0, c1 = 0, c2 = 0, c3 = 0;
  for (int base = s0; n_track && base < s1 && tstar < 0; base += 32) {
    const int i = base + lane;
    const int q = i < s1 ? quad[i] : 0;
    int a0 = q & 1, a1 = (q >> 1) & 1, a2 = (q >> 2) & 1, a3 = (q >> 3) & 1;
    for (int o = 1; o < 32; o <<= 1) {
      const int b0 = __shfl_up_sync(0xffffffffu, a0, o), b1 = __shfl_up_sync(0xffffffffu, a1, o);
      const int b2 = __shfl_up_sync(0xffffffffu, a2, o), b3 = __shfl_up_sync(0xffffffffu, a3, o);
      if (lane >= o) { a0 += b0; a1 += b1; a2 += b2; a3 += b3; }
    }
    a0 += c0; a1 += c1; a2 += c2; a3 += c3;
    const unsigned ok = __ballot_sync(0xffffffffu, i < s1 && a0 >= need && a1 >= need && a2 >= need && a3 >= need);
    if (ok) tstar = base + __ffs(ok) - 1;
    c0 = __shfl_sync(0xffffffffu, a0, 31); c1 = __shfl_sync(0xffffffffu, a1, 31);
    c2 = __shfl_sync(0xffffffffu, a2, 31); c3 = __shfl_sync(0xffffffffu, a3, 31);
  }
  if (lane == 0) {
    strength[v] = n_track == 0 ? newcnt[v] : (tstar < 0 ? 0 : s1 - tstar);
    in_table[v] = newcnt[v] > 0 || s1 > s0;
  }
}
// the table in ascending vertex order after the oldkey bump, and the LOCAL edges (other, newkey) of addNewEdges
__global__ void k_str_table(int V, int oldkey, int covis_thr, const int* __restrict__ in_table, const int* __restrict__ tptr,
                            int* __restrict__ strength, int* __restrict__ qual, int* __restrict__ rows) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  int s = strength[v];
  if (v == oldkey && s < covis_thr) s = covis_thr;   // slam_graph.cpp:172-175
  strength[v] = s;
  qual[v] = in_table[v] && s >= covis_thr;
  if (in_table[v]) { rows[2 * (size_t)tptr[v]] = v; rows[2 * (size_t)tptr[v] + 1] = s; }
}
__global__ void k_str_edges(int V, int newkey, const int* __restrict__ qual, const int* __restrict__ eptr,
                            const int* __restrict__ strength, int* __restrict__ v1, int* __restrict__ v2, int* __restrict__ es) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V || !qual[v]) return;
  v1[eptr[v]] = v; v2[eptr[v]] = newkey; es[eptr[v]] = strength[v];
}

// an edge of the request already in the graph, or a pair listed twice (insertEdge asserts, slam_graph.hpp:349-353)
__global__ void k_edge_exists(GraphDev g, int gV, int n, const int* __restrict__ v1, const int* __restrict__ v2, int* __restrict__ bad) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  if (v1[k] < gV && v2[k] < gV && has_edge(g, v1[k], v2[k])) atomicAdd(bad, 1);
}

// the feature tables (points in ascending id) of the vertices the new edges touch: flag, count, emit, sort
__global__ void k_touch(int n, const int* __restrict__ v1, const int* __restrict__ v2, int* __restrict__ touched) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) { touched[v1[k]] = 1; touched[v2[k]] = 1; }
}
__global__ void k_feat_count(MapDev m, const int* __restrict__ touched, int* __restrict__ fcnt) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= m.Np) return;
  for (int i = m.vis_ptr[p]; i < m.vis_ptr[p + 1]; ++i)
    if (touched[m.vis_pose[i]]) atomicAdd(fcnt + m.vis_pose[i], 1);
}
__global__ void k_feat_emit(MapDev m, const int* __restrict__ touched, const int* __restrict__ fptr, int* __restrict__ fcur,
                            unsigned long long* __restrict__ key) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= m.Np) return;
  for (int i = m.vis_ptr[p]; i < m.vis_ptr[p + 1]; ++i) {
    const int v = m.vis_pose[i];
    if (touched[v]) key[fptr[v] + atomicAdd(fcur + v, 1)] = (unsigned long long)v << 32 | (unsigned)p;
  }
}
__global__ void k_feat_unpack(int n, const unsigned long long* __restrict__ key, int* __restrict__ point) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) point[i] = (int)(unsigned)key[i];
}
__global__ void k_max(int n, const int* __restrict__ x, int* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicMax(out, x[i]);
}

// neighbour-list insertion.  Edge k inserts (strength[k], v2) into v1's list (sequence 2k) and then (strength[k], v1)
// into v2's (2k + 1), each as std::multimap::insert does (after the equal keys; lists are read through rbegin): in the
// stored order, strongest first, a new entry goes in front of the first entry with strength <= its own.
__global__ void k_ins_keys(int n, const int* __restrict__ v1, const int* __restrict__ v2, int* __restrict__ target,
                           int* __restrict__ seq, int* __restrict__ icnt) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= 2 * n) return;
  const int t = (j & 1) ? v2[j >> 1] : v1[j >> 1];
  target[j] = t; seq[j] = j;
  atomicAdd(icnt + t, 1);
}
__global__ void k_ins_count(int V, int gV, const int* __restrict__ old_ptr, const int* __restrict__ icnt, int* __restrict__ cnt) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) cnt[v] = (v < gV ? old_ptr[v + 1] - old_ptr[v] : 0) + icnt[v];
}
struct InsArgs {
  int n, gV, nn_old;
  GraphDev g;                     // the graph before the call (gV lists)
  const int *iptr, *iseq;         // the inserts grouped by target vertex, in sequence order inside a group
  const int *v1, *v2, *es;        // the edges
  const double *T12, *Lam;        // their constraints: T_1_from_2, Lambda
  const int* nptr;                // the new lists
  int *id, *str; double *T, *L; unsigned char* mrg;
};
__global__ void k_ins_move_old(InsArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.nn_old) return;
  int lo = 0, hi = a.gV;          // the vertex whose list holds entry i: nbr_ptr[v] <= i < nbr_ptr[v + 1]
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (a.g.nbr_ptr[mid] <= i) lo = mid; else hi = mid; }
  const int v = lo, s = a.g.nbr_str[i];
  int at = a.nptr[v] + (i - a.g.nbr_ptr[v]);
  for (int j = a.iptr[v]; j < a.iptr[v + 1]; ++j) at += a.es[a.iseq[j] >> 1] >= s;
  a.id[at] = a.g.nbr_id[i]; a.str[at] = s; a.mrg[at] = a.g.nbr_mrg[i];
  for (int q = 0; q < 7; ++q) a.T[7 * (size_t)at + q] = a.g.nbr_T[7 * (size_t)i + q];
  for (int q = 0; q < 36; ++q) a.L[36 * (size_t)at + q] = a.g.nbr_Lam[36 * (size_t)i + q];
}
__global__ void k_ins_move_new(InsArgs a, int V) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= 2 * a.n) return;
  const int sq = a.iseq[j], k = sq >> 1, s = a.es[k];
  int lo = 0, hi = V;             // the target vertex: iptr[v] <= j < iptr[v + 1]
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (a.iptr[mid] <= j) lo = mid; else hi = mid; }
  const int v = lo;
  int at = a.nptr[v];
  if (v < a.gV)
    for (int i = a.g.nbr_ptr[v]; i < a.g.nbr_ptr[v + 1]; ++i) at += a.g.nbr_str[i] > s;
  for (int r = a.iptr[v]; r < a.iptr[v + 1]; ++r) {
    const int s2 = a.es[a.iseq[r] >> 1];
    at += s2 > s || (s2 == s && a.iseq[r] > sq);
  }
  // setConstraint(v1, v2, T_1_from_2, Lambda, Lambda): v2's entry for v1 holds T_1_from_2, v1's entry its inverse
  a.id[at] = (sq & 1) ? a.v1[k] : a.v2[k]; a.str[at] = s; a.mrg[at] = 1;
  double Ti[7];
  const double* T12 = a.T12 + 7 * (size_t)k;
  if (!(sq & 1)) svs::se3_inv(T12, Ti);
  for (int q = 0; q < 7; ++q) a.T[7 * (size_t)at + q] = (sq & 1) ? T12[q] : Ti[q];
  for (int q = 0; q < 36; ++q) a.L[36 * (size_t)at + q] = a.Lam[36 * (size_t)k + q];
}

// ------------------------------------------------------------------ prepareForOptimization (slam_graph.cpp:290-310)
// reinitializePoses (:665-725).  The FIFO queue decides every vertex's parent, so one thread walks it as k_bfs does; a
// node carries its parent, the parent's entry for it (T_me_from_parent when the edge is marginalised) and the mark.
// Both skips happen at pop time.  The parent's pose is final once the parent has been popped.
struct ReinitNode { int v, parent, entry, mark; };
__global__ void k_reinit(GraphDev g, int root, int loop, const int* __restrict__ new_t, const int* __restrict__ old_t,
                         double* __restrict__ pose, int* __restrict__ seen, ReinitNode* __restrict__ queue, int qcap) {
  if (blockIdx.x || threadIdx.x) return;
  int head = 0, tail = 0;
  queue[tail++] = ReinitNode{root, -1, -1, 0};
  while (head < tail) {
    const ReinitNode n = queue[head++];
    if (seen[n.v] || !new_t[n.v]) continue;      // "Avoid cycles!", then "Skip is it is not in double window"
    seen[n.v] = 1;
    const int mark = n.mark || n.v == loop;
    if (n.parent >= 0 && (mark || !old_t[n.v])) {
      // T_me = getRelativePose_1_from_2(me, parent) * T_parent: the stored constraint of a marginalised edge, else
      // T_me * T_parent^-1 from the current poses
      double Tp[7], R[7], Pi[7], Tm[7];
      for (int q = 0; q < 7; ++q) { Tp[q] = pose[7 * (size_t)n.parent + q]; Tm[q] = pose[7 * (size_t)n.v + q]; }
      if (g.nbr_mrg[n.entry]) {
        for (int q = 0; q < 7; ++q) R[q] = g.nbr_T[7 * (size_t)n.entry + q];
      } else {
        svs::se3_inv(Tp, Pi);
        svs::se3_mul(Tm, Pi, R);
      }
      svs::se3_mul(R, Tp, Tm);
      for (int q = 0; q < 7; ++q) pose[7 * (size_t)n.v + q] = Tm[q];
    }
    for (int i = g.nbr_ptr[n.v]; i < g.nbr_ptr[n.v + 1] && tail < qcap; ++i) queue[tail++] = ReinitNode{g.nbr_id[i], n.v, i, mark};
  }
}

// margPosesLeftInnerWindow's pairs (:848-904): edges whose two ends were INNER in the old window and are not both INNER
// now, one row per edge from the entry of its larger end (v1 = max, v2 = min: the reference's second write wins);
// the vertices they touch get their feature tables
__device__ __forceinline__ bool leaves_inner(const int* old_t, const int* new_t, int a, int b) {
  return a > b && old_t[a] == 1 && old_t[b] == 1 && !(new_t[a] == 1 && new_t[b] == 1);
}
__global__ void k_marg_count(int V, GraphDev g, const int* __restrict__ old_t, const int* __restrict__ new_t, int* __restrict__ cnt,
                             int* __restrict__ touched) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= V) return;
  int c = 0;
  for (int i = g.nbr_ptr[a]; i < g.nbr_ptr[a + 1]; ++i) {
    const int b = g.nbr_id[i];
    if (leaves_inner(old_t, new_t, a, b)) { ++c; touched[b] = 1; }
  }
  cnt[a] = c;
  if (c) touched[a] = 1;
}
__global__ void k_marg_emit(int V, GraphDev g, const int* __restrict__ old_t, const int* __restrict__ new_t, const int* __restrict__ ptr,
                            int* __restrict__ v1, int* __restrict__ v2) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= V) return;
  int at = ptr[a];
  for (int i = g.nbr_ptr[a]; i < g.nbr_ptr[a + 1]; ++i)
    if (leaves_inner(old_t, new_t, a, g.nbr_id[i])) { v1[at] = a; v2[at] = g.nbr_id[i]; ++at; }
}
// unmargPosesEnteringInnerW (:728-759): an edge between two INNER frames of the new window is unmarginalised
__global__ void k_unmarg(int V, GraphDev g, const int* __restrict__ new_t, unsigned char* __restrict__ mrg) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= V || new_t[a] != 1) return;
  for (int i = g.nbr_ptr[a]; i < g.nbr_ptr[a + 1]; ++i)
    if (new_t[g.nbr_id[i]] == 1) mrg[i] = 0;
}
// setConstraint(v1, v2, T_1_from_2, Lambda, Lambda) on both entries of pair k, as k_ins_move_new stores a new edge
__global__ void k_marg_store(int n, GraphDev g, const int* __restrict__ v1, const int* __restrict__ v2, const double* __restrict__ T12,
                             const double* __restrict__ Lam, double* __restrict__ T, double* __restrict__ L, unsigned char* __restrict__ mrg) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  double Ti[7];
  svs::se3_inv(T12 + 7 * (size_t)k, Ti);
  for (int side = 0; side < 2; ++side) {
    const int me = side ? v1[k] : v2[k], nb = side ? v2[k] : v1[k];
    const double* t = side ? Ti : T12 + 7 * (size_t)k;
    for (int i = g.nbr_ptr[me]; i < g.nbr_ptr[me + 1]; ++i) {
      if (g.nbr_id[i] != nb) continue;
      for (int q = 0; q < 7; ++q) T[7 * (size_t)i + q] = t[q];
      for (int q = 0; q < 36; ++q) L[36 * (size_t)i + q] = Lam[36 * (size_t)k + q];
      mrg[i] = 1;
    }
  }
}

// the map's tables and the pose graph's lists, each carved from one device buffer; the handle keeps them writable
struct MapTables { double* pose; int* anchor; double* xyz; int* vis_ptr; int* vis_pose; double* center; int* level; };
MapTables map_carve(svs::Bump& m, int V, int Np, int nnz) {
  MapTables t;
  t.pose = m.take<double>(7 * (size_t)V); t.anchor = m.take<int>(Np); t.xyz = m.take<double>(3 * (size_t)Np);
  t.vis_ptr = m.take<int>((size_t)Np + 1); t.vis_pose = m.take<int>(nnz); t.center = m.take<double>(3 * (size_t)nnz);
  t.level = m.take<int>(nnz);
  return t;
}
struct GraphTables { int *ptr, *id, *str; double *T, *Lam; unsigned char* mrg; };
GraphTables graph_carve(svs::Bump& m, int V, int nn) {
  GraphTables t;
  t.ptr = m.take<int>((size_t)V + 1); t.id = m.take<int>(nn); t.str = m.take<int>(nn); t.T = m.take<double>(7 * (size_t)nn);
  t.Lam = m.take<double>(36 * (size_t)nn); t.mrg = m.take<unsigned char>(nn);
  return t;
}

}  // namespace

struct svs_map : svs::Handle {
  int V = 0, Np = 0, nnz = 0;
  char* d_map = nullptr; size_t map_cap = 0;
  MapTables t{}; MapDev m{};   // m: t as the kernels read it
  char* d_work = nullptr; size_t work_cap = 0;
  std::vector<int> h_winpos;
  const double* d_oi_last = nullptr;   // [E][3] observations, [E][3] weights of the last assembly
  const int* d_ep_last = nullptr; const int* d_es_last = nullptr; const int* d_ea_last = nullptr;   // its index triples
  int last_E = 0;
  // the last assembled window and the serial of the BA problem it became (svs::ba_problem_serial); d_win_last = nullptr
  // when there is none: the map was reloaded or grew, or the last assembly was refused
  const int* d_win_last = nullptr; const int* d_act_last = nullptr; int last_P = 0, last_L = 0;
  unsigned long long last_serial = 0;
  char* d_upd = nullptr; size_t upd_cap = 0;   // staging of svs_map_update_*
  char* d_graph = nullptr; size_t graph_cap = 0; GraphTables gt{}; GraphDev g{}; int nnzN = 0;   // svs_map_set_graph
  char* d_graph2 = nullptr; size_t graph2_cap = 0;   // the next graph while the growth calls build it (then swapped)
  char* d_gw = nullptr; size_t gw_cap = 0;           // work of the growth calls: strengths and staged edge lists
  char* d_ge = nullptr; size_t ge_cap = 0;           // ... feature tables, constraints and list insertion
  char* d_cs = nullptr; size_t cs_cap = 0;           // ... median scratch of the constraint kernel
  char* d_sel = nullptr; size_t sel_cap = 0;   // work buffers of svs_map_select_window / svs_map_prepare_for_optimization
  // the window of the last svs_map_prepare_for_optimization (0 / 1 INNER / 2 OUTER) for vertices [0, wtV); vertices
  // from wtV on (added since) are outside it.  wtV = 0: no window yet
  int* d_wt = nullptr; size_t wt_cap = 0; int wtV = 0;
};

static void map_bind(svs_map* h, const MapTables& t, int V, int Np, int nnz) {
  h->V = V; h->Np = Np; h->nnz = nnz;
  h->t = t;
  h->m = MapDev{V, Np, t.pose, t.anchor, t.xyz, t.vis_ptr, t.vis_pose, t.center, t.level};
}

extern "C" {

int svs_map_create(int device, svs_map** out) {
  if (!out) return SVS_ERR_INVALID;
  *out = nullptr;
  svs_map* h = new svs_map();
  if (int rc = svs::open_handle(h, device)) {
    delete h;
    return rc;
  }
  *out = h;
  return SVS_OK;
}

void svs_map_destroy(svs_map* h) {
  if (!h) return;
  svs::begin_close(h);
  cudaFree(h->d_map); cudaFree(h->d_work); cudaFree(h->d_upd); cudaFree(h->d_graph); cudaFree(h->d_sel);
  cudaFree(h->d_graph2); cudaFree(h->d_gw); cudaFree(h->d_ge); cudaFree(h->d_cs); cudaFree(h->d_wt);
  delete h;
}

const char* svs_map_last_error(const svs_map* h) { return svs::last_error(h); }

int svs_map_set(svs_map* h, int V, const double* T_me_from_world, int Np, const int* point_anchor, const double* xyz_anchor,
                const int* vis_ptr, const int* vis_pose, const double* feat_center, const int* feat_level) {
  if (!h || V <= 0 || Np < 0 || !T_me_from_world || (Np && (!point_anchor || !xyz_anchor || !vis_ptr))) return SVS_ERR_INVALID;
  const int nnz = Np ? vis_ptr[Np] : 0;
  if (nnz < 0 || (nnz && (!vis_pose || !feat_center || !feat_level))) return SVS_ERR_INVALID;
  for (int p = 0; p < Np; ++p) {
    if (point_anchor[p] < 0 || point_anchor[p] >= V) { h->err = "point anchored in a vertex outside [0, V)"; return SVS_ERR_INVALID; }
    if (vis_ptr[p + 1] < vis_ptr[p]) { h->err = "vis_ptr not ascending"; return SVS_ERR_INVALID; }
  }
  for (int i = 0; i < nnz; ++i)
    if (vis_pose[i] < 0 || vis_pose[i] >= V || feat_level[i] < 0 || feat_level[i] > 30) {
      h->err = "observation names a vertex outside [0, V) or a bad pyramid level";
      return SVS_ERR_INVALID;
    }
  cudaSetDevice(h->device);
  svs::Bump m{nullptr};
  map_carve(m, V, Np, nnz);
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  h->d_win_last = nullptr;   // a window assembled from the previous map names its rows, not this map's
  SVS_CK(h, svs::grow(m.off, &h->map_cap, &h->d_map));
  m = svs::Bump{h->d_map};
  const MapTables t = map_carve(m, V, Np, nnz);
  SVS_CK(h, cudaMemcpyAsync(t.pose, T_me_from_world, sizeof(double) * 7 * (size_t)V, cudaMemcpyHostToDevice, h->stream));
  if (Np) {
    SVS_CK(h, cudaMemcpyAsync(t.anchor, point_anchor, sizeof(int) * (size_t)Np, cudaMemcpyHostToDevice, h->stream));
    SVS_CK(h, cudaMemcpyAsync(t.xyz, xyz_anchor, sizeof(double) * 3 * (size_t)Np, cudaMemcpyHostToDevice, h->stream));
    SVS_CK(h, cudaMemcpyAsync(t.vis_ptr, vis_ptr, sizeof(int) * ((size_t)Np + 1), cudaMemcpyHostToDevice, h->stream));
  }
  if (nnz) {
    SVS_CK(h, cudaMemcpyAsync(t.vis_pose, vis_pose, sizeof(int) * (size_t)nnz, cudaMemcpyHostToDevice, h->stream));
    SVS_CK(h, cudaMemcpyAsync(t.center, feat_center, sizeof(double) * 3 * (size_t)nnz, cudaMemcpyHostToDevice, h->stream));
    SVS_CK(h, cudaMemcpyAsync(t.level, feat_level, sizeof(int) * (size_t)nnz, cudaMemcpyHostToDevice, h->stream));
  }
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  map_bind(h, t, V, Np, nnz);
  h->g = GraphDev{}; h->nnzN = 0; h->wtV = 0;   // a new map: its pose graph comes with svs_map_set_graph
  return SVS_OK;
}

// n records of `width` doubles go to the device in ONE copy and are scattered there
static int map_scatter(svs_map* h, double* table, int rows_in_table, int n, const int* index, const double* rows, int width,
                       const char* what) {
  for (int i = 0; i < n; ++i)
    if (index[i] < 0 || index[i] >= rows_in_table) { h->err = std::string(what) + " index out of range"; return SVS_ERR_INVALID; }
  if (n == 0) return SVS_OK;
  cudaSetDevice(h->device);
  int* d_index = nullptr; double* d_rows = nullptr;
  auto carve = [&](svs::Bump m) { d_index = m.take<int>(n); d_rows = m.take<double>((size_t)n * width); return m.off; };
  const size_t bytes = carve(svs::Bump{nullptr});
  if (bytes > h->upd_cap) {
    SVS_CK(h, cudaStreamSynchronize(h->stream));
    SVS_CK(h, svs::grow(bytes, &h->upd_cap, &h->d_upd));
  }
  carve(svs::Bump{h->d_upd});
  SVS_CK(h, cudaMemcpyAsync(d_index, index, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaMemcpyAsync(d_rows, rows, sizeof(double) * (size_t)n * width, cudaMemcpyHostToDevice, h->stream));
  k_scatter_rows<<<(n * width + 255) / 256, 256, 0, h->stream>>>(table, d_index, d_rows, n, width);
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaStreamSynchronize(h->stream));   // the caller's arrays may go away
  return SVS_OK;
}

int svs_map_update_poses(svs_map* h, int n, const int* vertex, const double* T_me_from_world) {
  if (!h || n < 0 || (n && (!vertex || !T_me_from_world)) || !h->d_map) return SVS_ERR_INVALID;
  return map_scatter(h, h->t.pose, h->V, n, vertex, T_me_from_world, 7, "vertex");
}

int svs_map_update_points(svs_map* h, int n, const int* point, const double* xyz_anchor) {
  if (!h || n < 0 || (n && (!point || !xyz_anchor)) || !h->d_map) return SVS_ERR_INVALID;
  return map_scatter(h, h->t.xyz, h->Np, n, point, xyz_anchor, 3, "point");
}

int svs_map_get(svs_map* h, double* T_me_from_world, double* xyz_anchor) {
  if (!h || !h->d_map) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  if (T_me_from_world) SVS_CK(h, cudaMemcpyAsync(T_me_from_world, h->m.pose, sizeof(double) * 7 * (size_t)h->V, cudaMemcpyDeviceToHost, h->stream));
  if (xyz_anchor && h->Np) SVS_CK(h, cudaMemcpyAsync(xyz_anchor, h->m.xyz, sizeof(double) * 3 * (size_t)h->Np, cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  return SVS_OK;
}

// SlamGraph::restoreDataFromG2o (slam_graph.cpp:1037-1058): the optimised window of `ba` (loaded with
// svs_ba_set_problem_from_map from THIS map) goes back into the map, device to device
int svs_map_absorb(svs_map* h, svs_ba* ba) {
  svs::NvtxRange nvtx_("restoreDataFromG2o");
  if (!h || !ba || !h->d_map) return SVS_ERR_INVALID;
  if (!h->d_win_last) { h->err = "no window of this map is waiting to be absorbed"; return SVS_ERR_STATE; }
  if (svs::ba_device(ba) != h->device) { h->err = "map and bundle adjuster live on different devices"; return SVS_ERR_INVALID; }
  const double* const* pose; const double* const* psi; const int* lm_user; const int* cur; cudaStream_t st; int P, L;
  if (svs::ba_state_on_device(ba, &pose, &psi, &lm_user, &cur, &st, &P, &L) != SVS_OK || P != h->last_P || L != h->last_L ||
      svs::ba_problem_serial(ba) != h->last_serial) {
    h->err = "the bundle adjuster does not hold the window this map assembled last";
    return SVS_ERR_STATE;
  }
  cudaSetDevice(h->device);
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  const int n = std::max(7 * P, L);
  k_absorb<<<(n + 255) / 256, 256, 0, st>>>(h->t.pose, h->t.xyz, pose[0], pose[1], psi[0], psi[1],
                                            lm_user, cur, h->d_win_last, h->d_act_last, P, L);
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaStreamSynchronize(st));
  return SVS_OK;
}

int svs_ba_set_problem_from_map(svs_ba* ba, svs_map* h, int P, const int* window_vertex, const unsigned char* fixed, int L,
                                const int* active_point, int C, const int* c_i, const int* c_j, const double* c_T,
                                const double* c_Lambda, const svs_cam* cam, int* num_edges) {
  svs::NvtxRange nvtx_("copyDataToG2o");
  if (!ba || !h || P <= 0 || L < 0 || C < 0 || !window_vertex || (L && !active_point) || !cam || !h->d_map) return SVS_ERR_INVALID;
  if (svs::ba_device(ba) != h->device) { h->err = "map and bundle adjuster live on different devices"; return SVS_ERR_INVALID; }
  h->d_win_last = nullptr;   // recorded again below once the BA handle has accepted this window
  if (C && (!c_i || !c_j || !c_T || !c_Lambda)) { h->err = "svs_ba_set_problem: null array"; return SVS_ERR_INVALID; }
  // window position of every vertex (-1 = outside the double window)
  h->h_winpos.assign(h->V, -1);
  for (int i = 0; i < P; ++i) {
    const int v = window_vertex[i];
    if (v < 0 || v >= h->V || h->h_winpos[v] >= 0) { h->err = "window names a vertex twice or outside [0, V)"; return SVS_ERR_INVALID; }
    h->h_winpos[v] = i;
  }
  for (int l = 0; l < L; ++l)
    if (active_point[l] < 0 || active_point[l] >= h->Np) { h->err = "active point outside [0, Np)"; return SVS_ERR_INVALID; }
  cudaSetDevice(h->device);
  // work arena: win_pos, window, active, cnt, ptr, bad | poses, psi | edges (sized for every observation of the map) |
  // the caller's fixed flags and pose-pose constraints (host arrays), next to the window
  struct {
    int *wp, *win, *act, *cnt, *ptr, *bad, *ep, *es, *ea, *ci, *cj; double *pose, *psi, *oi, *cT, *cL; unsigned char* fx;
  } w;
  auto carve = [&](svs::Bump m) {
    w.wp = m.take<int>(h->V); w.win = m.take<int>(P); w.act = m.take<int>(L); w.cnt = m.take<int>(L);
    w.ptr = m.take<int>((size_t)L + 1); w.bad = m.take<int>(1);
    w.pose = m.take<double>(7 * (size_t)P); w.psi = m.take<double>(3 * (size_t)L);
    w.ep = m.take<int>(h->nnz); w.es = m.take<int>(h->nnz); w.ea = m.take<int>(h->nnz); w.oi = m.take<double>(6 * (size_t)h->nnz);
    w.fx = m.take<unsigned char>(P); w.ci = m.take<int>(C); w.cj = m.take<int>(C);
    w.cT = m.take<double>(7 * (size_t)C); w.cL = m.take<double>(36 * (size_t)C);
    return m.off;
  };
  const size_t bytes = carve(svs::Bump{nullptr});
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  if (bytes > h->work_cap) {
    h->last_E = 0; h->d_oi_last = nullptr; h->d_ep_last = h->d_es_last = h->d_ea_last = nullptr;   // they lay in the old arena
    SVS_CK(h, svs::grow(bytes, &h->work_cap, &h->d_work));
  }
  carve(svs::Bump{h->d_work});
  SVS_CK(h, cudaMemcpyAsync(w.wp, h->h_winpos.data(), sizeof(int) * (size_t)h->V, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaMemcpyAsync(w.win, window_vertex, sizeof(int) * (size_t)P, cudaMemcpyHostToDevice, h->stream));
  if (L) SVS_CK(h, cudaMemcpyAsync(w.act, active_point, sizeof(int) * (size_t)L, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaMemsetAsync(w.bad, 0, sizeof(int), h->stream));
  if (fixed) SVS_CK(h, cudaMemcpyAsync(w.fx, fixed, (size_t)P, cudaMemcpyHostToDevice, h->stream));
  if (C) {
    SVS_CK(h, cudaMemcpyAsync(w.ci, c_i, sizeof(int) * (size_t)C, cudaMemcpyHostToDevice, h->stream));
    SVS_CK(h, cudaMemcpyAsync(w.cj, c_j, sizeof(int) * (size_t)C, cudaMemcpyHostToDevice, h->stream));
    SVS_CK(h, cudaMemcpyAsync(w.cT, c_T, sizeof(double) * 7 * (size_t)C, cudaMemcpyHostToDevice, h->stream));
    SVS_CK(h, cudaMemcpyAsync(w.cL, c_Lambda, sizeof(double) * 36 * (size_t)C, cudaMemcpyHostToDevice, h->stream));
  }
  int E = 0, bad = 0;
  if (L) {
    k_count<<<(L + 255) / 256, 256, 0, h->stream>>>(h->m, w.wp, w.act, L, w.cnt, w.bad);
    k_scan<<<1, 1024, 0, h->stream>>>(w.cnt, L, w.ptr);
    SVS_CK(h, cudaMemcpyAsync(&E, w.ptr + L, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    SVS_CK(h, cudaMemcpyAsync(&bad, w.bad, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    SVS_CK(h, cudaStreamSynchronize(h->stream));
    if (bad) { h->err = "an active point is anchored in a frame outside the window"; return SVS_ERR_INVALID; }
    // obs_info = [E][3] observations followed by [E][3] weights: the emit kernel needs E for the second half
    k_emit<<<(L + 255) / 256, 256, 0, h->stream>>>(h->m, w.wp, w.act, L, w.ptr, E, w.ep, w.es, w.ea, w.oi, w.psi);
  }
  k_gather_poses<<<(7 * P + 255) / 256, 256, 0, h->stream>>>(h->m, w.win, P, w.pose);
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaStreamSynchronize(h->stream));   // the BA handle reads the window on its own stream
  if (num_edges) *num_edges = E;
  h->d_oi_last = w.oi; h->last_E = E;
  h->d_ep_last = w.ep; h->d_es_last = w.es; h->d_ea_last = w.ea;
  // the window goes to the BA handle device to device: its structure is analysed there (svs_ba_set_problem_device)
  const int rc = svs::ba_set_problem_device_obs(ba, P, w.pose, fixed ? w.fx : nullptr, L, w.psi, E, w.ep, w.es,
                                                 w.ea, w.oi, C, w.ci, w.cj, w.cT, w.cL, cam);
  if (rc != SVS_OK) { h->err = std::string("svs_ba_set_problem: ") + svs_last_error(ba); return rc; }
  h->d_win_last = w.win; h->d_act_last = w.act; h->last_P = P; h->last_L = L;
  h->last_serial = svs::ba_problem_serial(ba);
  return SVS_OK;
}


// ------------------------------------------------------------------ pose graph, window selection, growth

static void graph_bind(svs_map* h, const GraphTables& t, int nn, bool strength, bool constraints) {
  h->gt = t;
  h->g = GraphDev{t.ptr, t.id, strength ? t.str : nullptr, constraints ? t.T : nullptr, constraints ? t.Lam : nullptr, t.mrg};
  h->nnzN = nn;
}

// pose_graph: the lists come with strengths and constraints (svs_map_set_pose_graph), all required when there are entries
static int upload_graph(svs_map* h, const int* nbr_ptr, const int* nbr_id, const int* nbr_strength, const double* nbr_T,
                        const double* nbr_Lambda, bool pose_graph) {
  if (!h || !h->d_map || !nbr_ptr) return SVS_ERR_INVALID;
  const int V = h->V, nn = nbr_ptr[V];
  if (nbr_ptr[0] != 0 || nn < 0 || (nn && !nbr_id) || ((nbr_T == nullptr) != (nbr_Lambda == nullptr))) return SVS_ERR_INVALID;
  if (pose_graph && nn && (!nbr_strength || !nbr_T)) return SVS_ERR_INVALID;
  for (int v = 0; v < V; ++v)
    if (nbr_ptr[v + 1] < nbr_ptr[v]) { h->err = "nbr_ptr not ascending"; return SVS_ERR_INVALID; }
  for (int i = 0; i < nn; ++i)
    if (nbr_id[i] < 0 || nbr_id[i] >= V) { h->err = "neighbour outside [0, V)"; return SVS_ERR_INVALID; }
  if (pose_graph)
    for (int v = 0; v < V; ++v)
      for (int i = nbr_ptr[v] + 1; i < nbr_ptr[v + 1]; ++i)
        if (nbr_strength[i] > nbr_strength[i - 1]) { h->err = "a neighbour list is not ordered strongest first"; return SVS_ERR_INVALID; }
  cudaSetDevice(h->device);
  svs::Bump m{nullptr};
  graph_carve(m, V, nn);
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  SVS_CK(h, svs::grow(m.off, &h->graph_cap, &h->d_graph));
  m = svs::Bump{h->d_graph};
  const GraphTables t = graph_carve(m, V, nn);
  SVS_CK(h, cudaMemcpyAsync(t.ptr, nbr_ptr, sizeof(int) * ((size_t)V + 1), cudaMemcpyHostToDevice, h->stream));
  if (nn) {
    SVS_CK(h, cudaMemcpyAsync(t.id, nbr_id, sizeof(int) * (size_t)nn, cudaMemcpyHostToDevice, h->stream));
    if (pose_graph) SVS_CK(h, cudaMemcpyAsync(t.str, nbr_strength, sizeof(int) * (size_t)nn, cudaMemcpyHostToDevice, h->stream));
    if (nbr_T) {
      SVS_CK(h, cudaMemcpyAsync(t.T, nbr_T, sizeof(double) * 7 * (size_t)nn, cudaMemcpyHostToDevice, h->stream));
      SVS_CK(h, cudaMemcpyAsync(t.Lam, nbr_Lambda, sizeof(double) * 36 * (size_t)nn, cudaMemcpyHostToDevice, h->stream));
    }
  }
  // the reference's state at its first prepareForOptimization: addNewEdges and addLoopClosure end in setConstraint
  SVS_CK(h, cudaMemsetAsync(t.mrg, 1, (size_t)std::max(nn, 1), h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  graph_bind(h, t, nn, pose_graph, pose_graph || nbr_T != nullptr);
  h->wtV = 0;
  return SVS_OK;
}

int svs_map_set_graph(svs_map* h, const int* nbr_ptr, const int* nbr_id, const double* nbr_T, const double* nbr_Lambda) {
  return upload_graph(h, nbr_ptr, nbr_id, nullptr, nbr_T, nbr_Lambda, false);
}

int svs_map_set_pose_graph(svs_map* h, const int* nbr_ptr, const int* nbr_id, const int* nbr_strength, const double* nbr_T,
                           const double* nbr_Lambda) {
  return upload_graph(h, nbr_ptr, nbr_id, nbr_strength, nbr_T, nbr_Lambda, true);
}

int svs_map_get_graph(svs_map* h, int cap, int* nnzN, int* nbr_ptr, int* nbr_id, int* nbr_strength, double* nbr_T,
                      double* nbr_Lambda) {
  if (!h || !h->d_map || !nnzN) return SVS_ERR_INVALID;
  if (!h->g.nbr_ptr) { h->err = "the map has no pose graph"; return SVS_ERR_STATE; }
  const int V = h->V, nn = h->nnzN;
  *nnzN = nn;
  if ((nbr_id || nbr_strength || nbr_T || nbr_Lambda) && cap < nn) { h->err = "nnzN exceeds the caller's capacity"; return SVS_ERR_INVALID; }
  cudaSetDevice(h->device);
  if (nbr_ptr) SVS_CK(h, cudaMemcpyAsync(nbr_ptr, h->g.nbr_ptr, sizeof(int) * ((size_t)V + 1), cudaMemcpyDeviceToHost, h->stream));
  if (nn) {
    if (nbr_id) SVS_CK(h, cudaMemcpyAsync(nbr_id, h->g.nbr_id, sizeof(int) * (size_t)nn, cudaMemcpyDeviceToHost, h->stream));
    if (nbr_strength && h->g.nbr_str)
      SVS_CK(h, cudaMemcpyAsync(nbr_strength, h->g.nbr_str, sizeof(int) * (size_t)nn, cudaMemcpyDeviceToHost, h->stream));
    if (nbr_T && h->g.nbr_T) SVS_CK(h, cudaMemcpyAsync(nbr_T, h->g.nbr_T, sizeof(double) * 7 * (size_t)nn, cudaMemcpyDeviceToHost, h->stream));
    if (nbr_Lambda && h->g.nbr_Lam)
      SVS_CK(h, cudaMemcpyAsync(nbr_Lambda, h->g.nbr_Lam, sizeof(double) * 36 * (size_t)nn, cudaMemcpyDeviceToHost, h->stream));
  }
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  // what the graph does not hold reads as strength 0, the identity and Lambda = 0 (as svs_map_select_window pairs it)
  for (int i = 0; i < nn; ++i) {
    if (nbr_strength && !h->g.nbr_str) nbr_strength[i] = 0;
    if (nbr_T && !h->g.nbr_T) for (int q = 0; q < 7; ++q) nbr_T[7 * (size_t)i + q] = q == 3 ? 1. : 0.;
    if (nbr_Lambda && !h->g.nbr_Lam) memset(nbr_Lambda + 36 * (size_t)i, 0, sizeof(double) * 36);
  }
  return SVS_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ window selection (svs_map_select_window and prepare)
struct SelWork { int *type, *ext, *wtype, *flag, *ptrV, *win, *pos, *act, *ptrP, *actl, *q, *cc, *cp, *ci, *cj; double *cT, *cL; };
static SelWork sel_carve(svs::Bump& m, int V, int Np, int nn) {
  SelWork s;
  s.type = m.take<int>(V); s.ext = m.take<int>(V); s.wtype = m.take<int>(V); s.flag = m.take<int>(V);
  s.ptrV = m.take<int>((size_t)V + 1); s.win = m.take<int>(V); s.pos = m.take<int>(V); s.act = m.take<int>(Np);
  s.ptrP = m.take<int>((size_t)Np + 1); s.actl = m.take<int>(Np); s.q = m.take<int>((size_t)nn + 1); s.cc = m.take<int>(V);
  s.cp = m.take<int>((size_t)V + 1); s.ci = m.take<int>(nn); s.cj = m.take<int>(nn); s.cT = m.take<double>(7 * (size_t)nn);
  s.cL = m.take<double>(36 * (size_t)nn);
  return s;
}

// computeInitialDoubleWin + computeActivePointsAndExtendOuterWindow and the pair count of copyContraintsToG2o, enqueued
// on the map's stream; the counts P, L, C go to counts[0..2] once the stream is synchronised.  The window types (0 / 1
// INNER / 2 OUTER) are left in s.wtype.
static int sel_enqueue(svs_map* h, const SelWork& s, int root, int inner, int dbl, int* counts) {
  const int V = h->V, Np = h->Np, nn = h->nnzN;
  SVS_CK(h, cudaMemsetAsync(s.type, 0, sizeof(int) * V, h->stream));
  SVS_CK(h, cudaMemsetAsync(s.ext, 0, sizeof(int) * V, h->stream));
  const int bV = (V + 255) / 256, bP = (std::max(Np, 1) + 255) / 256;
  k_bfs<<<1, 32, 0, h->stream>>>(V, h->g, root, inner, dbl, s.type, s.q, nn + 1);
  if (Np) k_active<<<bP, 256, 0, h->stream>>>(h->m, h->g, s.type, s.ext, s.act);
  k_window_flags<<<bV, 256, 0, h->stream>>>(V, s.type, s.ext, s.wtype, s.flag);
  k_scan<<<1, 1024, 0, h->stream>>>(s.flag, V, s.ptrV);
  k_compact<<<bV, 256, 0, h->stream>>>(V, s.flag, s.ptrV, s.win, s.pos);
  if (Np) {
    k_scan<<<1, 1024, 0, h->stream>>>(s.act, Np, s.ptrP);
    k_compact<<<bP, 256, 0, h->stream>>>(Np, s.act, s.ptrP, s.actl, nullptr);
  }
  k_pair_count<<<bV, 256, 0, h->stream>>>(V, h->g, s.wtype, s.cc);
  k_scan<<<1, 1024, 0, h->stream>>>(s.cc, V, s.cp);
  SVS_CK(h, cudaGetLastError());
  counts[1] = 0;
  SVS_CK(h, cudaMemcpyAsync(counts, s.ptrV + V, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  if (Np) SVS_CK(h, cudaMemcpyAsync(counts + 1, s.ptrP + Np, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaMemcpyAsync(counts + 2, s.cp + V, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  return SVS_OK;
}

// the window's outputs once the counts fit: the pairs with the graph's constraints as they are now, then the copies
static int sel_emit(svs_map* h, const SelWork& s, int P, int L, int C, int* window_vertex, unsigned char* inner,
                    int* active_point, int* c_i, int* c_j, double* c_T, double* c_Lambda) {
  const int V = h->V;
  k_pair_emit<<<(V + 255) / 256, 256, 0, h->stream>>>(V, h->g, s.wtype, s.pos, s.cp, s.ci, s.cj, s.cT, s.cL);
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaMemcpyAsync(window_vertex, s.win, sizeof(int) * (size_t)P, cudaMemcpyDeviceToHost, h->stream));
  if (L) SVS_CK(h, cudaMemcpyAsync(active_point, s.actl, sizeof(int) * (size_t)L, cudaMemcpyDeviceToHost, h->stream));
  h->h_winpos.resize(V);
  SVS_CK(h, cudaMemcpyAsync(h->h_winpos.data(), s.wtype, sizeof(int) * (size_t)V, cudaMemcpyDeviceToHost, h->stream));
  if (c_i && C) {
    if (!c_j || !c_T || !c_Lambda) return SVS_ERR_INVALID;
    SVS_CK(h, cudaMemcpyAsync(c_i, s.ci, sizeof(int) * (size_t)C, cudaMemcpyDeviceToHost, h->stream));
    SVS_CK(h, cudaMemcpyAsync(c_j, s.cj, sizeof(int) * (size_t)C, cudaMemcpyDeviceToHost, h->stream));
    SVS_CK(h, cudaMemcpyAsync(c_T, s.cT, sizeof(double) * 7 * (size_t)C, cudaMemcpyDeviceToHost, h->stream));
    SVS_CK(h, cudaMemcpyAsync(c_Lambda, s.cL, sizeof(double) * 36 * (size_t)C, cudaMemcpyDeviceToHost, h->stream));
  }
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  if (inner)
    for (int i = 0; i < P; ++i) inner[i] = h->h_winpos[window_vertex[i]] == 1;
  return SVS_OK;
}

static bool sel_args_ok(int cap_P, int* P_out, int* window_vertex, int cap_L, int* L_out, int* active_point, int cap_C) {
  return P_out && window_vertex && L_out && (!cap_L || active_point) && cap_P > 0 && cap_L >= 0 && cap_C >= 0;
}

extern "C" int svs_map_select_window(svs_map* h, int root, int inner_window_size, int double_window_size, int cap_P, int* P_out,
                                     int* window_vertex, unsigned char* inner, int cap_L, int* L_out, int* active_point, int cap_C,
                                     int* C_out, int* c_i, int* c_j, double* c_T, double* c_Lambda) {
  if (!h || !h->d_map || !sel_args_ok(cap_P, P_out, window_vertex, cap_L, L_out, active_point, cap_C)) return SVS_ERR_INVALID;
  if (!h->g.nbr_ptr) { h->err = "svs_map_set_graph has not been called for this map"; return SVS_ERR_STATE; }
  const int V = h->V;
  if (root < 0 || root >= V || inner_window_size < 0 || inner_window_size >= double_window_size) {   // assert at slam_graph.cpp:563
    h->err = "root outside [0, V) or inner_window_size >= double_window_size";
    return SVS_ERR_INVALID;
  }
  cudaSetDevice(h->device);
  svs::Bump m{nullptr};
  sel_carve(m, V, h->Np, h->nnzN);
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  SVS_CK(h, svs::grow(m.off, &h->sel_cap, &h->d_sel));
  m = svs::Bump{h->d_sel};
  const SelWork s = sel_carve(m, V, h->Np, h->nnzN);
  int counts[3] = {0, 0, 0};
  if (int rc = sel_enqueue(h, s, root, inner_window_size, double_window_size, counts)) return rc;
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  const int P = counts[0], L = counts[1], C = counts[2];
  *P_out = P; *L_out = L;
  if (C_out) *C_out = C;
  if (P > cap_P || L > cap_L || (c_i && C > cap_C)) { h->err = "window, active points or constraints exceed the caller's capacity"; return SVS_ERR_INVALID; }
  return sel_emit(h, s, P, L, C, window_vertex, inner, active_point, c_i, c_j, c_T, c_Lambda);
}


static int keyframe_check(svs_map* h, int oldkey, const double* T_newkey_from_oldkey, int n_new, const int* new_anchor,
                          const double* new_xyz_anchor, const double* new_anchor_center, const int* new_anchor_level,
                          const double* new_center, const int* new_level, int n_track, const int* track_point,
                          const double* track_center, const int* track_level) {
  if (!h || !h->d_map || !T_newkey_from_oldkey || n_new < 0 || n_track < 0 ||
      (n_new && (!new_anchor || !new_xyz_anchor || !new_anchor_center || !new_anchor_level || !new_center || !new_level)) ||
      (n_track && (!track_point || !track_center || !track_level)))
    return SVS_ERR_INVALID;
  const int V = h->V, Np = h->Np;
  if (oldkey < 0 || oldkey >= V) { h->err = "oldkey outside [0, V)"; return SVS_ERR_INVALID; }
  for (int q = 0; q < n_new; ++q)
    if (new_anchor[q] < 0 || new_anchor[q] >= V || new_anchor_level[q] < 0 || new_anchor_level[q] > 30 || new_level[q] < 0 || new_level[q] > 30) {
      h->err = "new point anchored outside [0, V) or bad pyramid level";
      return SVS_ERR_INVALID;
    }
  {
    std::vector<int> tp(track_point, track_point + n_track);
    std::sort(tp.begin(), tp.end());
    for (int t = 0; t < n_track; ++t)
      if (tp[t] < 0 || tp[t] >= Np || (t && tp[t] == tp[t - 1]) || track_level[t] < 0 || track_level[t] > 30) {
        h->err = "tracked point outside [0, Np), listed twice, or bad pyramid level";
        return SVS_ERR_INVALID;
      }
  }
  return SVS_OK;
}

// the growth of svs_map_add_keyframe on checked arguments; the pose graph is left as it was
static int keyframe_grow(svs_map* h, int oldkey, const double* T_newkey_from_oldkey, int n_new, const int* new_anchor,
                         const double* new_xyz_anchor, const double* new_anchor_center, const int* new_anchor_level,
                         const double* new_center, const int* new_level, int n_track, const int* track_point,
                         const double* track_center, const int* track_level) {
  const int V = h->V, Np = h->Np, nnz = h->nnz;
  cudaSetDevice(h->device);
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  const int V2 = V + 1, Np2 = Np + n_new, nnz2 = nnz + n_track + 2 * n_new;
  svs::Bump mz{nullptr};
  map_carve(mz, V2, Np2, nnz2);
  const size_t cap = mz.off + mz.off / 4;
  char* B2 = nullptr;
  SVS_CK(h, cudaMalloc(&B2, cap));
  svs::Bump mb{B2};
  const MapTables t = map_carve(mb, V2, Np2, nnz2);
  // staging: everything the kernels read from the caller, carved alike in a host vector and the device buffer so that
  // one pinned-less copy (keyframe rate, a few 10 KB) moves the prefix [0, up); add and cnt are the kernels' own
  struct Stage { double *T, *nx, *nac, *nc, *tc; int *na, *nal, *nl, *tp, *tl, *add, *cnt; size_t up, end; };
  auto carve = [&](char* base) {
    svs::Bump m{base};
    Stage g;
    g.T = m.take<double>(7); g.na = m.take<int>(n_new); g.nx = m.take<double>(3 * (size_t)n_new);
    g.nac = m.take<double>(3 * (size_t)n_new); g.nal = m.take<int>(n_new); g.nc = m.take<double>(3 * (size_t)n_new);
    g.nl = m.take<int>(n_new); g.tp = m.take<int>(n_track); g.tc = m.take<double>(3 * (size_t)n_track);
    g.tl = m.take<int>(n_track);
    g.up = m.off;
    g.add = m.take<int>(Np2); g.cnt = m.take<int>(Np2);
    g.end = m.off;
    return g;
  };
  std::vector<char> st(carve(nullptr).end);
  const Stage hs = carve(st.data());
  auto put = [](void* dst, const void* src, size_t bytes) { if (bytes) memcpy(dst, src, bytes); };
  put(hs.T, T_newkey_from_oldkey, sizeof(double) * 7);
  put(hs.na, new_anchor, sizeof(int) * (size_t)n_new); put(hs.nx, new_xyz_anchor, sizeof(double) * 3 * (size_t)n_new);
  put(hs.nac, new_anchor_center, sizeof(double) * 3 * (size_t)n_new); put(hs.nal, new_anchor_level, sizeof(int) * (size_t)n_new);
  put(hs.nc, new_center, sizeof(double) * 3 * (size_t)n_new); put(hs.nl, new_level, sizeof(int) * (size_t)n_new);
  put(hs.tp, track_point, sizeof(int) * (size_t)n_track); put(hs.tc, track_center, sizeof(double) * 3 * (size_t)n_track);
  put(hs.tl, track_level, sizeof(int) * (size_t)n_track);
  if (svs::grow(st.size(), &h->upd_cap, &h->d_upd) != cudaSuccess) { cudaFree(B2); h->err = "cudaMalloc"; return SVS_ERR_CUDA; }
  const Stage u = carve(h->d_upd);
  cudaError_t e = cudaMemcpyAsync(h->d_upd, st.data(), u.up, cudaMemcpyHostToDevice, h->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(u.add, 0xff, sizeof(int) * (size_t)Np2, h->stream);
  // vertices
  if (e == cudaSuccess) e = cudaMemcpyAsync(t.pose, h->m.pose, sizeof(double) * 7 * (size_t)V, cudaMemcpyDeviceToDevice, h->stream);
  k_new_pose<<<1, 32, 0, h->stream>>>(h->m.pose, oldkey, u.T, t.pose + 7 * (size_t)V);
  // points
  if (Np && e == cudaSuccess) e = cudaMemcpyAsync(t.anchor, h->m.anchor, sizeof(int) * (size_t)Np, cudaMemcpyDeviceToDevice, h->stream);
  if (Np && e == cudaSuccess) e = cudaMemcpyAsync(t.xyz, h->m.xyz, sizeof(double) * 3 * (size_t)Np, cudaMemcpyDeviceToDevice, h->stream);
  if (n_new && e == cudaSuccess) e = cudaMemcpyAsync(t.anchor + Np, u.na, sizeof(int) * (size_t)n_new, cudaMemcpyDeviceToDevice, h->stream);
  if (n_new && e == cudaSuccess) e = cudaMemcpyAsync(t.xyz + 3 * (size_t)Np, u.nx, sizeof(double) * 3 * (size_t)n_new, cudaMemcpyDeviceToDevice, h->stream);
  // observations
  if (Np2) {
    if (n_track) k_mark_tracks<<<(n_track + 255) / 256, 256, 0, h->stream>>>(n_track, u.tp, u.add);
    k_grow_count<<<(Np2 + 255) / 256, 256, 0, h->stream>>>(h->m, Np2, V, u.add, u.cnt);
    k_scan<<<1, 1024, 0, h->stream>>>(u.cnt, Np2, t.vis_ptr);
    k_grow_move<<<(Np2 + 255) / 256, 256, 0, h->stream>>>(h->m, Np2, V, u.add, t.vis_ptr, u.tc, u.tl, u.na, u.nac, u.nal, u.nc,
                                                        u.nl, t.vis_pose, t.center, t.level);
  }
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e != cudaSuccess) { cudaFree(B2); h->err = std::string("svs_map_add_keyframe: ") + cudaGetErrorString(e); return SVS_ERR_CUDA; }
  cudaFree(h->d_map);
  h->d_map = B2; h->map_cap = cap;
  map_bind(h, t, V2, Np2, nnz2);
  h->d_win_last = nullptr;                 // (a window assembled before the growth can no longer be absorbed)
  return SVS_OK;
}

extern "C" int svs_map_add_keyframe(svs_map* h, int oldkey, const double* T_newkey_from_oldkey, int n_new, const int* new_anchor,
                                    const double* new_xyz_anchor, const double* new_anchor_center, const int* new_anchor_level,
                                    const double* new_center, const int* new_level, int n_track, const int* track_point,
                                    const double* track_center, const int* track_level, int* vertex_index,
                                    int* first_new_point) {
  int rc = keyframe_check(h, oldkey, T_newkey_from_oldkey, n_new, new_anchor, new_xyz_anchor, new_anchor_center, new_anchor_level,
                          new_center, new_level, n_track, track_point, track_center, track_level);
  const int V = rc == SVS_OK ? h->V : 0, Np = rc == SVS_OK ? h->Np : 0;
  if (rc == SVS_OK)
    rc = keyframe_grow(h, oldkey, T_newkey_from_oldkey, n_new, new_anchor, new_xyz_anchor, new_anchor_center, new_anchor_level,
                       new_center, new_level, n_track, track_point, track_center, track_level);
  if (rc != SVS_OK) return rc;
  h->g = GraphDev{}; h->nnzN = 0; h->wtV = 0;   // the pose graph changed with the new vertex: svs_map_set_graph again
  if (vertex_index) *vertex_index = V;
  if (first_new_point) *first_new_point = Np;
  return SVS_OK;
}

// The feature tables (points in ascending id) of the vertices flagged in `touched`, for computeConstraint.  Clear,
// flag, count (nfeat and the largest table go to ctl[0], ctl[1]), then -- once the caller has read ctl on the host --
// build: emit one key (vertex, point) per observation, sort with CUB, unpack into point.
struct FeatWork { int *touch, *fcnt, *fptr, *fcur, *ctl, *fpt; unsigned long long *fkey, *fkey2; };
static FeatWork feat_carve(svs::Bump& m, int V, size_t nf) {
  FeatWork f;
  f.touch = m.take<int>(V); f.fcnt = m.take<int>(V); f.fptr = m.take<int>((size_t)V + 1); f.fcur = m.take<int>(V);
  f.ctl = m.take<int>(4); f.fkey = m.take<unsigned long long>(nf); f.fkey2 = m.take<unsigned long long>(nf);
  f.fpt = m.take<int>(nf);
  return f;
}
static size_t feat_sort_bytes(size_t nf) {
  size_t b = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, b, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)nf);
  return b;
}
static cudaError_t feat_clear(svs_map* h, const FeatWork& f) {
  cudaError_t e = cudaSuccess;
  for (int* p : {f.touch, f.fcnt, f.fcur})
    if (e == cudaSuccess) e = cudaMemsetAsync(p, 0, sizeof(int) * h->V, h->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(f.ctl, 0, sizeof(int) * 4, h->stream);
  return e;
}
static cudaError_t feat_count(svs_map* h, const FeatWork& f) {
  const int V = h->V, Np = h->Np;
  if (Np) k_feat_count<<<(Np + 255) / 256, 256, 0, h->stream>>>(h->m, f.touch, f.fcnt);
  k_scan<<<1, 1024, 0, h->stream>>>(f.fcnt, V, f.fptr);
  k_max<<<(V + 255) / 256, 256, 0, h->stream>>>(V, f.fcnt, f.ctl + 1);
  return cudaMemcpyAsync(f.ctl, f.fptr + V, sizeof(int), cudaMemcpyDeviceToDevice, h->stream);
}
static cudaError_t feat_build(svs_map* h, const FeatWork& f, int nfeat, void* tmp, size_t tmp_bytes) {
  if (!nfeat) return cudaSuccess;
  k_feat_emit<<<(h->Np + 255) / 256, 256, 0, h->stream>>>(h->m, f.touch, f.fptr, f.fcur, f.fkey);
  cudaError_t e = cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, f.fkey, f.fkey2, nfeat, 0, 64, h->stream);
  k_feat_unpack<<<(nfeat + 255) / 256, 256, 0, h->stream>>>(nfeat, f.fkey2, f.fpt);
  return e;
}

// addNewEdges' list insertion and setConstraint for n edges (device arrays v1, v2, strength on the map's stream):
// the feature tables of the vertices they touch, computeConstraint(v1, v2) on `poses` (the map's, or a copy with one
// vertex moved), then the new lists with their constraints.  The graph before the call has gV <= V lists; the lists of
// vertices gV..V-1 start empty.
static int grow_graph(svs_map* h, int gV, int n, const int* d_v1, const int* d_v2, const int* d_es, const double* d_poses) {
  const int V = h->V, nn_old = h->nnzN, nn = nn_old + 2 * n;
  const size_t nf = (size_t)std::max(h->nnz, 1), ni = (size_t)std::max(2 * n, 1);
  cudaSetDevice(h->device);
  size_t tmp_bytes = feat_sort_bytes(nf), b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b, (int*)nullptr, (int*)nullptr, (int*)nullptr, (int*)nullptr, (int)ni);
  tmp_bytes = std::max(tmp_bytes, b);
  FeatWork f;
  struct { double *T12, *Lam; int *cs, *icnt, *iptr, *ncnt, *tgt, *tgt2, *seq, *seq2; char* tmp; } w;
  auto carve = [&](svs::Bump m) {
    f = feat_carve(m, V, nf);
    w.T12 = m.take<double>(7 * ni); w.Lam = m.take<double>(36 * ni); w.cs = m.take<int>(ni);
    w.icnt = m.take<int>(V); w.iptr = m.take<int>((size_t)V + 1); w.ncnt = m.take<int>(V);
    w.tgt = m.take<int>(ni); w.tgt2 = m.take<int>(ni); w.seq = m.take<int>(ni); w.seq2 = m.take<int>(ni);
    w.tmp = m.take<char>(tmp_bytes);
    return m.off;
  };
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  SVS_CK(h, svs::grow(carve(svs::Bump{nullptr}), &h->ge_cap, &h->d_ge));
  carve(svs::Bump{h->d_ge});
  svs::Bump m{nullptr};
  graph_carve(m, V, nn);
  SVS_CK(h, svs::grow(m.off, &h->graph2_cap, &h->d_graph2));
  m = svs::Bump{h->d_graph2};
  const GraphTables t = graph_carve(m, V, nn);
  const int bV = (V + 255) / 256;
  SVS_CK(h, feat_clear(h, f));
  SVS_CK(h, cudaMemsetAsync(w.icnt, 0, sizeof(int) * V, h->stream));
  if (n) {
    k_touch<<<(n + 255) / 256, 256, 0, h->stream>>>(n, d_v1, d_v2, f.touch);
    SVS_CK(h, feat_count(h, f));
    int ctl[2] = {0, 0};
    SVS_CK(h, cudaMemcpyAsync(ctl, f.ctl, sizeof(int) * 2, cudaMemcpyDeviceToHost, h->stream));
    SVS_CK(h, cudaStreamSynchronize(h->stream));
    const int nfeat = ctl[0], stride = svs::constraint_scratch_stride(ctl[1]);
    SVS_CK(h, feat_build(h, f, nfeat, w.tmp, tmp_bytes));
    if (stride) {
      SVS_CK(h, cudaStreamSynchronize(h->stream));
      SVS_CK(h, svs::grow(sizeof(double) * (size_t)stride * n, &h->cs_cap, &h->d_cs));
    }
    svs::launch_compute_constraint(d_poses, f.fptr, f.fpt, h->m.anchor, h->m.xyz, n, d_v1, d_v2, w.T12, w.Lam, w.cs,
                                   reinterpret_cast<double*>(h->d_cs), stride, h->stream);
    k_ins_keys<<<(2 * n + 255) / 256, 256, 0, h->stream>>>(n, d_v1, d_v2, w.tgt, w.seq, w.icnt);
    size_t tb = tmp_bytes;   // a stable sort: inside one target the inserts stay in sequence order
    SVS_CK(h, cub::DeviceRadixSort::SortPairs(w.tmp, tb, w.tgt, w.tgt2, w.seq, w.seq2, 2 * n, 0, 32, h->stream));
  }
  k_scan<<<1, 1024, 0, h->stream>>>(w.icnt, V, w.iptr);
  k_ins_count<<<bV, 256, 0, h->stream>>>(V, gV, h->g.nbr_ptr, w.icnt, w.ncnt);
  k_scan<<<1, 1024, 0, h->stream>>>(w.ncnt, V, t.ptr);
  InsArgs a;
  a.n = n; a.gV = gV; a.nn_old = nn_old; a.g = h->g; a.iptr = w.iptr; a.iseq = w.seq2;
  a.v1 = d_v1; a.v2 = d_v2; a.es = d_es; a.T12 = w.T12; a.Lam = w.Lam;
  a.nptr = t.ptr; a.id = t.id; a.str = t.str; a.T = t.T; a.L = t.Lam; a.mrg = t.mrg;
  if (nn_old) k_ins_move_old<<<(nn_old + 255) / 256, 256, 0, h->stream>>>(a);
  if (n) k_ins_move_new<<<(2 * n + 255) / 256, 256, 0, h->stream>>>(a, V);
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  std::swap(h->d_graph, h->d_graph2); std::swap(h->graph_cap, h->graph2_cap);
  graph_bind(h, t, nn, true, true);
  return SVS_OK;
}

static int needs_pose_graph(svs_map* h) {
  if (!h->g.nbr_ptr || !h->g.nbr_str || !h->g.nbr_T) {
    h->err = "the map has no pose graph with strengths and constraints (svs_map_set_pose_graph)";
    return SVS_ERR_STATE;
  }
  return SVS_OK;
}

extern "C" int svs_map_add_keyframe_graph(svs_map* h, int oldkey, const double* T_newkey_from_oldkey, int n_new,
                                          const int* new_anchor, const double* new_xyz_anchor, const double* new_anchor_center,
                                          const int* new_anchor_level, const double* new_center, const int* new_level,
                                          int n_track, const int* track_point, const double* track_center,
                                          const int* track_level, int covis_thr, int width, int height, int* vertex_index,
                                          int* first_new_point, int* n_table, int* table, int* n_edges) {
  svs::NvtxRange nvtx_("addKeyframe");
  int rc = keyframe_check(h, oldkey, T_newkey_from_oldkey, n_new, new_anchor, new_xyz_anchor, new_anchor_center, new_anchor_level,
                          new_center, new_level, n_track, track_point, track_center, track_level);
  if (rc != SVS_OK) return rc;
  if (covis_thr < 1 || width <= 0 || height <= 0) { h->err = "covis_thr < 1 or an empty image"; return SVS_ERR_INVALID; }
  if ((rc = needs_pose_graph(h)) != SVS_OK) return rc;
  const int V = h->V, Np = h->Np;
  const size_t nr = (size_t)std::max(h->nnz, 1);   // records: the tracked points are distinct, so at most nnz
  cudaSetDevice(h->device);
  size_t tmp_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (unsigned char*)nullptr, (unsigned char*)nullptr, (int)nr);
  struct {
    int *tp, *na, *tcnt, *tptr, *vcnt, *vptr, *nw, *str, *in, *rptr, *qual, *eptr, *rows, *v1, *v2, *es;
    double* tc; unsigned long long *key, *key2; unsigned char *q, *q2; char* tmp;
  } w;
  auto carve = [&](svs::Bump m) {
    w.tp = m.take<int>(n_track); w.tc = m.take<double>(3 * (size_t)n_track); w.na = m.take<int>(n_new);
    w.tcnt = m.take<int>(n_track); w.tptr = m.take<int>((size_t)n_track + 1);
    w.vcnt = m.take<int>(V); w.vptr = m.take<int>((size_t)V + 1); w.nw = m.take<int>(V);
    w.str = m.take<int>(V); w.in = m.take<int>(V); w.rptr = m.take<int>((size_t)V + 1);
    w.qual = m.take<int>(V); w.eptr = m.take<int>((size_t)V + 1); w.rows = m.take<int>(2 * (size_t)V);
    w.v1 = m.take<int>(V); w.v2 = m.take<int>(V); w.es = m.take<int>(V);
    w.key = m.take<unsigned long long>(nr); w.key2 = m.take<unsigned long long>(nr);
    w.q = m.take<unsigned char>(nr); w.q2 = m.take<unsigned char>(nr); w.tmp = m.take<char>(tmp_bytes);
    return m.off;
  };
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  SVS_CK(h, svs::grow(carve(svs::Bump{nullptr}), &h->gw_cap, &h->d_gw));
  carve(svs::Bump{h->d_gw});
  if (n_track) {
    SVS_CK(h, cudaMemcpyAsync(w.tp, track_point, sizeof(int) * n_track, cudaMemcpyHostToDevice, h->stream));
    SVS_CK(h, cudaMemcpyAsync(w.tc, track_center, sizeof(double) * 3 * n_track, cudaMemcpyHostToDevice, h->stream));
  }
  if (n_new) SVS_CK(h, cudaMemcpyAsync(w.na, new_anchor, sizeof(int) * n_new, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaMemsetAsync(w.vcnt, 0, sizeof(int) * V, h->stream));
  SVS_CK(h, cudaMemsetAsync(w.nw, 0, sizeof(int) * V, h->stream));
  // computeStrength on the map before the growth
  int R = 0;
  if (n_track) {
    k_str_count<<<(n_track + 255) / 256, 256, 0, h->stream>>>(h->m, n_track, w.tp, w.tcnt);
    k_scan<<<1, 1024, 0, h->stream>>>(w.tcnt, n_track, w.tptr);
    SVS_CK(h, cudaMemcpyAsync(&R, w.tptr + n_track, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    SVS_CK(h, cudaStreamSynchronize(h->stream));
  }
  if (R) {
    const int half_w = (int)(width * 0.5), half_h = (int)(height * 0.5);   // int half_width = cam_.width()*0.5 (:480-481)
    k_str_emit<<<(n_track + 255) / 256, 256, 0, h->stream>>>(h->m, n_track, w.tp, w.tc, (double)half_w, (double)half_h, w.tptr,
                                                             w.key, w.q, w.vcnt);
    size_t tb = tmp_bytes;
    SVS_CK(h, cub::DeviceRadixSort::SortPairs(w.tmp, tb, w.key, w.key2, w.q, w.q2, R, 0, 64, h->stream));
  }
  if (n_new) k_str_new<<<(n_new + 255) / 256, 256, 0, h->stream>>>(n_new, w.na, w.nw);
  const int bV = (V + 255) / 256;
  k_scan<<<1, 1024, 0, h->stream>>>(w.vcnt, V, w.vptr);
  k_str_closed<<<(int)((32 * (size_t)V + 255) / 256), 256, 0, h->stream>>>(V, n_track, std::max(1, covis_thr / 2), w.vptr, w.q2,
                                                                          w.nw, w.str, w.in);
  k_scan<<<1, 1024, 0, h->stream>>>(w.in, V, w.rptr);
  k_str_table<<<bV, 256, 0, h->stream>>>(V, oldkey, covis_thr, w.in, w.rptr, w.str, w.qual, w.rows);
  k_scan<<<1, 1024, 0, h->stream>>>(w.qual, V, w.eptr);
  k_str_edges<<<bV, 256, 0, h->stream>>>(V, V, w.qual, w.eptr, w.str, w.v1, w.v2, w.es);
  SVS_CK(h, cudaGetLastError());
  int rows = 0, ne = 0, old_in = 0;
  SVS_CK(h, cudaMemcpyAsync(&rows, w.rptr + V, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaMemcpyAsync(&ne, w.eptr + V, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaMemcpyAsync(&old_in, w.in + oldkey, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  if (!old_in) { h->err = "oldkey is absent from the strength table (slam_graph.cpp:165 asserts)"; return SVS_ERR_INVALID; }
  if (table && rows) SVS_CK(h, cudaMemcpyAsync(table, w.rows, sizeof(int) * 2 * (size_t)rows, cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  // addNewPointsToMap + addNewObsToOldPoints, then addNewEdges(LOCAL) on the grown map
  if ((rc = keyframe_grow(h, oldkey, T_newkey_from_oldkey, n_new, new_anchor, new_xyz_anchor, new_anchor_center, new_anchor_level,
                          new_center, new_level, n_track, track_point, track_center, track_level)) != SVS_OK)
    return rc;
  if ((rc = grow_graph(h, V, ne, w.v1, w.v2, w.es, h->m.pose)) != SVS_OK) {
    h->g = GraphDev{}; h->nnzN = 0; h->wtV = 0;   // the map has V + 1 vertices now: a graph of V lists must not stay behind
    return rc;
  }
  if (vertex_index) *vertex_index = V;
  if (first_new_point) *first_new_point = Np;
  if (n_table) *n_table = rows;
  if (n_edges) *n_edges = ne;
  return SVS_OK;
}

extern "C" int svs_map_add_edges(svs_map* h, int n, const int* v1, const int* v2, const int* strength, int moved_vertex,
                                 const double* T_moved_from_w) {
  if (!h || !h->d_map || n < 0 || (n && (!v1 || !v2 || !strength))) return SVS_ERR_INVALID;
  int rc = needs_pose_graph(h);
  if (rc != SVS_OK) return rc;
  const int V = h->V;
  if (moved_vertex < -1 || moved_vertex >= V || (moved_vertex >= 0 && !T_moved_from_w)) {
    h->err = "moved_vertex outside [-1, V) or its pose missing";
    return SVS_ERR_INVALID;
  }
  std::vector<std::pair<int, int>> pairs(n);
  for (int k = 0; k < n; ++k) {
    if (v1[k] < 0 || v1[k] >= V || v2[k] < 0 || v2[k] >= V || v1[k] == v2[k]) {
      h->err = "an edge names a vertex outside [0, V) or joins a vertex to itself";
      return SVS_ERR_INVALID;
    }
    pairs[k] = {std::min(v1[k], v2[k]), std::max(v1[k], v2[k])};
  }
  std::sort(pairs.begin(), pairs.end());
  if (std::adjacent_find(pairs.begin(), pairs.end()) != pairs.end()) { h->err = "an edge is listed twice"; return SVS_ERR_INVALID; }
  if (n == 0) return SVS_OK;
  cudaSetDevice(h->device);
  int *d_v1 = nullptr, *d_v2 = nullptr, *d_es = nullptr, *d_bad = nullptr; double* d_pose = nullptr;
  auto carve = [&](svs::Bump m) {
    d_v1 = m.take<int>(n); d_v2 = m.take<int>(n); d_es = m.take<int>(n); d_bad = m.take<int>(1); d_pose = m.take<double>(7 * (size_t)V);
    return m.off;
  };
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  SVS_CK(h, svs::grow(carve(svs::Bump{nullptr}), &h->gw_cap, &h->d_gw));
  carve(svs::Bump{h->d_gw});
  SVS_CK(h, cudaMemcpyAsync(d_v1, v1, sizeof(int) * n, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaMemcpyAsync(d_v2, v2, sizeof(int) * n, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaMemcpyAsync(d_es, strength, sizeof(int) * n, cudaMemcpyHostToDevice, h->stream));
  SVS_CK(h, cudaMemsetAsync(d_bad, 0, sizeof(int), h->stream));
  k_edge_exists<<<(n + 255) / 256, 256, 0, h->stream>>>(h->g, V, n, d_v1, d_v2, d_bad);
  SVS_CK(h, cudaGetLastError());
  int bad = 0;
  SVS_CK(h, cudaMemcpyAsync(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  if (bad) { h->err = "an edge is already in the pose graph (insertEdge asserts, slam_graph.hpp:353)"; return SVS_ERR_INVALID; }
  // registerKeyframes / addLoopClosure place the moved vertex at its new pose while the constraints are computed
  const double* poses = h->m.pose;
  if (moved_vertex >= 0) {
    SVS_CK(h, cudaMemcpyAsync(d_pose, h->m.pose, sizeof(double) * 7 * V, cudaMemcpyDeviceToDevice, h->stream));
    SVS_CK(h, cudaMemcpyAsync(d_pose + 7 * (size_t)moved_vertex, T_moved_from_w, sizeof(double) * 7, cudaMemcpyHostToDevice, h->stream));
    poses = d_pose;
  }
  return grow_graph(h, V, n, d_v1, d_v2, d_es, poses);
}

// ------------------------------------------------------------------ prepareForOptimization
struct PrepWork {
  SelWork s; FeatWork f;
  int *old, *seen, *mcnt, *mptr, *v1, *v2, *cs; ReinitNode* q; double *T12, *Lam; char* tmp;
};

// steps 2, 4 and 5 once the counts have fitted: from here on the map changes
static int prepare_apply(svs_map* h, const PrepWork& w, int root, int loop, int P, int nM, int nfeat, int max_feat) {
  const int V = h->V, nn = h->nnzN;
  const int* new_t = w.s.wtype;
  h->d_win_last = nullptr;   // absorbing the previous window would overwrite the reinitialised poses
  SVS_CK(h, cudaMemsetAsync(w.seen, 0, sizeof(int) * V, h->stream));
  k_reinit<<<1, 32, 0, h->stream>>>(h->g, root, loop, new_t, w.old, h->t.pose, w.seen, w.q, nn + 1);
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  SVS_CK(h, svs::grow(sizeof(int) * (size_t)V, &h->wt_cap, &h->d_wt));
  SVS_CK(h, cudaMemcpyAsync(h->d_wt, new_t, sizeof(int) * (size_t)V, cudaMemcpyDeviceToDevice, h->stream));
  h->wtV = V;
  if (P >= 2) {
    const int bV = (V + 255) / 256;
    k_unmarg<<<bV, 256, 0, h->stream>>>(V, h->g, new_t, h->gt.mrg);
    if (nM) {
      k_marg_emit<<<bV, 256, 0, h->stream>>>(V, h->g, w.old, new_t, w.mptr, w.v1, w.v2);
      SVS_CK(h, feat_build(h, w.f, nfeat, w.tmp, feat_sort_bytes((size_t)std::max(h->nnz, 1))));
      const int stride = svs::constraint_scratch_stride(max_feat);
      if (stride) {
        SVS_CK(h, cudaStreamSynchronize(h->stream));
        SVS_CK(h, svs::grow(sizeof(double) * (size_t)stride * nM, &h->cs_cap, &h->d_cs));
      }
      // computeConstraint(v1 = max, v2 = min) at the reinitialised poses
      svs::launch_compute_constraint(h->m.pose, w.f.fptr, w.f.fpt, h->m.anchor, h->m.xyz, nM, w.v1, w.v2, w.T12, w.Lam, w.cs,
                                     reinterpret_cast<double*>(h->d_cs), stride, h->stream);
      k_marg_store<<<(nM + 255) / 256, 256, 0, h->stream>>>(nM, h->g, w.v1, w.v2, w.T12, w.Lam, h->gt.T, h->gt.Lam, h->gt.mrg);
    }
  }
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  return SVS_OK;
}

extern "C" int svs_map_prepare_for_optimization(svs_map* h, int root, int loop, int inner_window_size, int double_window_size,
                                                int* do_optimization, int cap_P, int* P_out, int* window_vertex,
                                                unsigned char* inner, int cap_L, int* L_out, int* active_point, int cap_C,
                                                int* C_out, int* c_i, int* c_j, double* c_T, double* c_Lambda) {
  svs::NvtxRange nvtx_("prepareForOptimization");
  if (!h || !h->d_map || !do_optimization || !sel_args_ok(cap_P, P_out, window_vertex, cap_L, L_out, active_point, cap_C))
    return SVS_ERR_INVALID;
  int rc = needs_pose_graph(h);
  if (rc != SVS_OK) return rc;
  const int V = h->V, nn = h->nnzN;
  if (root < 0 || root >= V || loop < -1 || loop >= V || inner_window_size < 0 || inner_window_size >= double_window_size) {
    h->err = "root outside [0, V), loop outside [-1, V) or inner_window_size >= double_window_size";
    return SVS_ERR_INVALID;
  }
  cudaSetDevice(h->device);
  const size_t nf = (size_t)std::max(h->nnz, 1);
  PrepWork w;
  auto carve = [&](svs::Bump m) {
    w.s = sel_carve(m, V, h->Np, nn);
    w.f = feat_carve(m, V, nf);
    w.old = m.take<int>(V); w.seen = m.take<int>(V); w.q = m.take<ReinitNode>((size_t)nn + 1);
    w.mcnt = m.take<int>(V); w.mptr = m.take<int>((size_t)V + 1); w.v1 = m.take<int>(nn); w.v2 = m.take<int>(nn);
    w.T12 = m.take<double>(7 * (size_t)nn); w.Lam = m.take<double>(36 * (size_t)nn); w.cs = m.take<int>(nn);
    w.tmp = m.take<char>(feat_sort_bytes(nf));
    return m.off;
  };
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  SVS_CK(h, svs::grow(carve(svs::Bump{nullptr}), &h->sel_cap, &h->d_sel));
  carve(svs::Bump{h->d_sel});
  // every count the call needs, before anything changes: window, active points, pairs, marginalised edges, features
  SVS_CK(h, cudaMemsetAsync(w.old, 0, sizeof(int) * V, h->stream));   // vertices from wtV on are outside the old window
  if (h->wtV) SVS_CK(h, cudaMemcpyAsync(w.old, h->d_wt, sizeof(int) * (size_t)h->wtV, cudaMemcpyDeviceToDevice, h->stream));
  int counts[6] = {0, 0, 0, 0, 0, 0};
  if ((rc = sel_enqueue(h, w.s, root, inner_window_size, double_window_size, counts)) != SVS_OK) return rc;
  SVS_CK(h, feat_clear(h, w.f));
  k_marg_count<<<(V + 255) / 256, 256, 0, h->stream>>>(V, h->g, w.old, w.s.wtype, w.mcnt, w.f.touch);
  k_scan<<<1, 1024, 0, h->stream>>>(w.mcnt, V, w.mptr);
  SVS_CK(h, feat_count(h, w.f));
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaMemcpyAsync(counts + 3, w.mptr + V, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaMemcpyAsync(counts + 4, w.f.ctl, sizeof(int) * 2, cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  const int P = counts[0], L = counts[1], C = counts[2];
  *P_out = P; *L_out = L;
  if (C_out) *C_out = C;
  *do_optimization = P >= 2;
  if (P > cap_P || L > cap_L || (c_i && C > cap_C)) { h->err = "window, active points or constraints exceed the caller's capacity"; return SVS_ERR_INVALID; }
  if ((rc = prepare_apply(h, w, root, loop, P, counts[3], counts[4], counts[5])) != SVS_OK) {
    h->g = GraphDev{}; h->nnzN = 0; h->wtV = 0;   // a graph half marginalised must not stay behind
    return rc;
  }
  return sel_emit(h, w.s, P, L, C, window_vertex, inner, active_point, c_i, c_j, c_T, c_Lambda);
}

extern "C" int svs_map_get_window_state(svs_map* h, int cap, int* nnzN, unsigned char* window_type, unsigned char* marginalized) {
  if (!h || !h->d_map || !nnzN) return SVS_ERR_INVALID;
  if (!h->g.nbr_ptr) { h->err = "the map has no pose graph"; return SVS_ERR_STATE; }
  const int V = h->V, nn = h->nnzN;
  *nnzN = nn;
  if (marginalized && cap < nn) { h->err = "nnzN exceeds the caller's capacity"; return SVS_ERR_INVALID; }
  cudaSetDevice(h->device);
  std::vector<int> wt(h->wtV);
  if (window_type && h->wtV)
    SVS_CK(h, cudaMemcpyAsync(wt.data(), h->d_wt, sizeof(int) * (size_t)h->wtV, cudaMemcpyDeviceToHost, h->stream));
  if (marginalized && nn) SVS_CK(h, cudaMemcpyAsync(marginalized, h->g.nbr_mrg, (size_t)nn, cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  if (window_type)
    for (int v = 0; v < V; ++v) window_type[v] = (unsigned char)(v < h->wtV ? wt[v] : 0);
  return SVS_OK;
}

extern "C" {

// the assembled edge list of the last svs_ba_set_problem_from_map, for inspection
int svs_map_last_edges(svs_map* h, int E, int* e_point, int* e_pose, int* e_anchor, double* e_obs, double* e_info) {
  if (!h || E != h->last_E || !h->d_work) return SVS_ERR_INVALID;
  if (E == 0) return SVS_OK;
  cudaSetDevice(h->device);
  if (e_point) SVS_CK(h, cudaMemcpy(e_point, h->d_ep_last, sizeof(int) * (size_t)E, cudaMemcpyDeviceToHost));
  if (e_pose) SVS_CK(h, cudaMemcpy(e_pose, h->d_es_last, sizeof(int) * (size_t)E, cudaMemcpyDeviceToHost));
  if (e_anchor) SVS_CK(h, cudaMemcpy(e_anchor, h->d_ea_last, sizeof(int) * (size_t)E, cudaMemcpyDeviceToHost));
  if (e_obs) SVS_CK(h, cudaMemcpy(e_obs, h->d_oi_last, sizeof(double) * 3 * (size_t)E, cudaMemcpyDeviceToHost));
  if (e_info) SVS_CK(h, cudaMemcpy(e_info, h->d_oi_last + 3 * (size_t)E, sizeof(double) * 3 * (size_t)E, cudaMemcpyDeviceToHost));
  return SVS_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ hooks of loop.cu (internal.cuh)

void svs::map_view(svs_map* h, MapView* v) {
  v->V = h->V; v->Np = h->Np; v->nnz = h->nnz; v->device = h->device; v->stream = h->stream; v->base = h;
  v->pose = h->m.pose; v->anchor = h->m.anchor; v->xyz = h->m.xyz; v->vis_ptr = h->m.vis_ptr; v->vis_pose = h->m.vis_pose;
  v->center = h->m.center; v->level = h->m.level;
}

bool svs::map_graph(svs_map* h, const int** nbr_ptr, const int** nbr_id, int* nnzN) {
  *nbr_ptr = h->g.nbr_ptr; *nbr_id = h->g.nbr_id; *nnzN = h->nnzN;
  return h->g.nbr_ptr != nullptr;
}

void svs::launch_scan(const int* cnt, int n, int* ptr, cudaStream_t stream) { k_scan<<<1, 1024, 0, stream>>>(cnt, n, ptr); }

int svs::map_add_observations(svs_map* h, int vertex, int n, const int* d_point, const double* d_center, const int* d_level) {
  const int V = h->V, Np = h->Np, nnz = h->nnz;
  if (n == 0 || Np == 0) return SVS_OK;
  cudaSetDevice(h->device);
  // the new tables are sized for n more observations (the handle keeps their pointers: nothing lays them out again);
  // nnz becomes what the scan counted (a point the vertex already observes gains none)
  int *add = nullptr, *cnt = nullptr;
  auto carve = [&](svs::Bump m) { add = m.take<int>(Np); cnt = m.take<int>(Np); return m.off; };
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  SVS_CK(h, svs::grow(carve(svs::Bump{nullptr}), &h->upd_cap, &h->d_upd));
  carve(svs::Bump{h->d_upd});
  svs::Bump mz{nullptr};
  map_carve(mz, V, Np, nnz + n);
  const size_t cap = mz.off + mz.off / 4;
  char* B2 = nullptr;
  SVS_CK(h, cudaMalloc(&B2, cap));
  svs::Bump mb{B2};
  const MapTables t = map_carve(mb, V, Np, nnz + n);
  int nnz2 = 0;
  cudaError_t e = cudaMemsetAsync(add, 0xff, sizeof(int) * (size_t)Np, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(t.pose, h->m.pose, sizeof(double) * 7 * (size_t)V, cudaMemcpyDeviceToDevice, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(t.anchor, h->m.anchor, sizeof(int) * (size_t)Np, cudaMemcpyDeviceToDevice, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(t.xyz, h->m.xyz, sizeof(double) * 3 * (size_t)Np, cudaMemcpyDeviceToDevice, h->stream);
  if (e == cudaSuccess) {
    k_mark_tracks<<<(n + 255) / 256, 256, 0, h->stream>>>(n, d_point, add);
    k_grow_count<<<(Np + 255) / 256, 256, 0, h->stream>>>(h->m, Np, vertex, add, cnt);
    k_scan<<<1, 1024, 0, h->stream>>>(cnt, Np, t.vis_ptr);
    k_grow_move<<<(Np + 255) / 256, 256, 0, h->stream>>>(h->m, Np, vertex, add, t.vis_ptr, d_center, d_level, nullptr, nullptr,
                                                        nullptr, nullptr, nullptr, t.vis_pose, t.center, t.level);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(&nnz2, t.vis_ptr + Np, sizeof(int), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e != cudaSuccess) { cudaFree(B2); h->err = std::string("map_add_observations: ") + cudaGetErrorString(e); return SVS_ERR_CUDA; }
  cudaFree(h->d_map);
  h->d_map = B2; h->map_cap = cap;
  map_bind(h, t, V, Np, nnz2);
  h->d_win_last = nullptr;   // the window's observations changed; the pose graph (V vertices) stays
  return SVS_OK;
}
