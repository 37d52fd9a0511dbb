// loop.cu -- metric verification of a proposed loop on sm_90a: Backend::globalLoopClosure (scavislam/backend.cpp:830-1001)
// with matchAndAlign (:726-784) from the device map, the matcher's keyframe slots and the motion-only LM, and the
// commit of SlamGraph::addLoopClosure's addNewObsToOldPoints on the loop vertex (slam_graph.cpp:220, 400-420); and the
// re-registration of a keyframe against the frames of its neighbourhood, Backend::localRegisterFrame (:549-784) with
// SlamGraph::registerKeyframes' addNewObsToOldPoints on the root vertex (slam_graph.cpp:189-205, 400-420).
//
// Kernels of this file: the candidate scan (points a vertex set observes: flag / scan / compact over the map, then
// test / scan / emit over those), the slot-pose refresh, the one-CTA loop gate, and for the registration the bounded
// neighbourhood BFS, the gate with its per-vertex counts, the stats table and the commit selection.  Matching, the LM
// and the observation commit run in match.cu, pose.cu and graph.cu.  The projections are compiled with -fmad=false and written operation by
// operation like oracle/loop_oracle.c, so that the (int) frame test and the gate agree with it bit for bit.
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/svs_b200.h"
#include "internal.cuh"
#include "se3_dev.cuh"
#include "svs_nvtx.hpp"

namespace {

constexpr int kGate = 256;   // the gate's CTA

struct Pose7 { double v[7]; };
struct Cam4 { double f, px, py, b; };
struct Levels { int w[SVS_MATCH_MAX_LEVELS], h[SVS_MATCH_MAX_LEVELS]; double f[SVS_MATCH_MAX_LEVELS], px[SVS_MATCH_MAX_LEVELS], py[SVS_MATCH_MAX_LEVELS]; int n; };

// the control word: device-side findings and the counts and poses the host reads back
struct LoopCtl {
  double T_loop_from_w[7];
  double T_newloop_from_w[7];
  int no_anchor_obs, bad_level, no_slot;
  int n_matched;
  int n_tracks, num_left, num_right, num_upper, num_lower;
  int n_direct, n_neighborhood, n_neighbors;   // localRegisterFrame
  double T_newroot_from_w[7];
};

__device__ __forceinline__ void se3_act(const double A[7], const double x[3], double y[3]) {
  double R[9];
  svs::quat_to_R(A, R);
  svs::mat3_vec(R, x, y);
  y[0] += A[4]; y[1] += A[5]; y[2] += A[6];
}

// T_loop_from_world = T_query_from_loop^-1 * T_query_from_world (backend.cpp:844-845)
__global__ void k_loop_setup(const double* __restrict__ map_pose, int query, Pose7 Tql, LoopCtl* ctl) {
  if (blockIdx.x || threadIdx.x) return;
  double Tlq[7];
  svs::se3_inv(Tql.v, Tlq);
  svs::se3_mul(Tlq, map_pose + 7 * (size_t)query, ctl->T_loop_from_w);
}

// a point is flagged when a vertex of the set vset[V] observes it
__global__ void k_query_flag(svs::MapView m, const int* __restrict__ vset, int* __restrict__ flag) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= m.Np) return;
  int f = 0;
  for (int i = m.vis_ptr[p]; i < m.vis_ptr[p + 1]; ++i) f |= vset[m.vis_pose[i]];
  flag[p] = f;
}

__global__ void k_compact_ids(int n, const int* __restrict__ flag, const int* __restrict__ ptr, int* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flag[i]) out[ptr[i]] = i;
}

// the candidate test of backend.cpp:853-893 / :493-535 for the nq flagged points (qpts, ascending), projected into the
// reference frame T_ref_from_w (device memory)
__global__ void k_cand_test(svs::MapView m, const int* __restrict__ qpts, const int* __restrict__ qptr, const int* __restrict__ inwin,
                            const int* __restrict__ slot, Levels lv, const double* __restrict__ T_ref_from_w, LoopCtl* ctl,
                            int* __restrict__ cflag,
                            svs_match_point* __restrict__ rec) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= qptr[m.Np]) return;
  const int p = qpts[i];
  const int a = m.anchor[p];
  cflag[i] = 0;
  if (!inwin[a]) return;
  int ia = -1;
  for (int k = m.vis_ptr[p]; k < m.vis_ptr[p + 1] && ia < 0; ++k)
    if (m.vis_pose[k] == a) ia = k;
  if (ia < 0) { atomicOr(&ctl->no_anchor_obs, 1); return; }
  const int l = m.level[ia];
  if (l >= lv.n) { atomicOr(&ctl->bad_level, 1); return; }
  double Twa[7], Tla[7], x[3];
  svs::se3_inv(m.pose + 7 * (size_t)a, Twa);
  svs::se3_mul(T_ref_from_w, Twa, Tla);
  se3_act(Tla, m.xyz + 3 * (size_t)p, x);
  const double u = lv.f[l] * (x[0] / x[2]) + lv.px[l];
  const double v = lv.f[l] * (x[1] / x[2]) + lv.py[l];
  const int ui = (int)u, vi = (int)v;
  if (!(ui >= 0 && ui < lv.w[l] && vi >= 0 && vi < lv.h[l])) return;
  if (slot[a] < 0) { atomicOr(&ctl->no_slot, 1); return; }
  svs_match_point r;
  r.keyframe = slot[a];
  r.anchor_level = l;
  const double s = (double)(1 << l);
  r.anchor_obs_pyr[0] = m.center[3 * (size_t)ia] / s;       // the inverse of slam_graph.cpp:387-389
  r.anchor_obs_pyr[1] = m.center[3 * (size_t)ia + 1] / s;
  for (int k = 0; k < 3; ++k) r.xyz_anchor[k] = m.xyz[3 * (size_t)p + k];
  rec[i] = r;
  cflag[i] = 1;
}

__global__ void k_cand_emit(int Np, const int* __restrict__ qptr, const int* __restrict__ qpts, const int* __restrict__ cflag,
                            const int* __restrict__ cptr, const svs_match_point* __restrict__ rec, svs_match_point* __restrict__ pts,
                            int* __restrict__ cpoint) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= qptr[Np] || !cflag[i]) return;
  pts[cptr[i]] = rec[i];
  cpoint[cptr[i]] = qpts[i];
}

// save (dir 0) or restore (dir 1) the pose of every slot
__global__ void k_slot_copy(int nslot, double* __restrict__ slot_T, size_t stride, double* __restrict__ save, int dir) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 7 * nslot) return;
  double* t = reinterpret_cast<double*>(reinterpret_cast<char*>(slot_T) + (size_t)(i / 7) * stride) + i % 7;
  if (dir) *t = save[i]; else save[i] = *t;
}

// the reference's vertex_table: every slot gets its vertex's map pose, the slot of vertex `over` (-1: none) T_over.
// Only the device copy of the slot poses changes; the matcher's host mirror keeps the poses last set through the C ABI.
// That is safe as long as the matcher uploads a slot's record only right after setting that slot's pose
// (svs_matcher_set_keyframe, svs_matcher_set_pyramid_device), which is how match.cu does it.
__global__ void k_slot_refresh(int V, const double* __restrict__ map_pose, const int* __restrict__ slot, int over,
                               const double* __restrict__ T_over, double* __restrict__ slot_T, size_t stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 7 * V) return;
  const int v = i / 7, q = i % 7;
  if (slot[v] < 0) return;
  double* t = reinterpret_cast<double*>(reinterpret_cast<char*>(slot_T) + (size_t)slot[v] * stride);
  t[q] = v == over ? T_over[q] : map_pose[7 * (size_t)v + q];
}

__global__ void __launch_bounds__(kGate) k_count_matched(const svs_match_result* __restrict__ res, int n, LoopCtl* ctl) {
  __shared__ int s;
  if (threadIdx.x == 0) s = 0;
  __syncthreads();
  int c = 0;
  for (int i = threadIdx.x; i < n; i += kGate) c += res[i].matched;
  atomicAdd(&s, c);
  __syncthreads();
  if (threadIdx.x == 0) ctl->n_matched = s;
}

// the reprojection test of backend.cpp:929-935 / :635-641: within 2 * 2^level pixels in u and v and within 6 in u_right
__device__ __forceinline__ bool gate_keep(const svs_match_result& r, const double R[9], const double T[7], const Cam4& cam, int lvl) {
  const int factor = 1 << lvl;   // zeroFromPyr_i(1, level)
  return svs::reproj_gate(r, R, T, cam.f, cam.px, cam.py, cam.b, 2.0 * factor, 2.0 * 3);
}

// backend.cpp:904-961 in one CTA: reproject each match with T_newloop_from_oldloop (SE3XYZ_STEREO::map as k_pose_lm
// computes it), keep it within the thresholds, count the quadrants and compact the kept ones in match order
__global__ void __launch_bounds__(kGate) k_gate(const svs_match_result* __restrict__ res, const svs_match_point* __restrict__ pts,
                                                const int* __restrict__ cpoint, int n, Pose7 T, Pose7 Tql, Cam4 cam, int w0, int h0,
                                                const double* __restrict__ map_pose, int query, LoopCtl* ctl,
                                                int* __restrict__ track_point, double* __restrict__ track_uvu,
                                                int* __restrict__ track_level) {
  __shared__ int sw[kGate / 32];
  __shared__ int carry;
  __shared__ int quad[4];
  if (threadIdx.x < 4) quad[threadIdx.x] = 0;
  if (threadIdx.x == 0) carry = 0;
  double R[9];
  svs::quat_to_R(T.v, R);
  int left = 0, right = 0, upper = 0, lower = 0;
  __syncthreads();
  for (int base = 0; base < n; base += kGate) {
    const int i = base + threadIdx.x;
    int keep = 0;
    double ob[3] = {0, 0, 0};
    int lvl = 0;
    if (i < n && res[i].matched) {
      const svs_match_result& r = res[i];
      ob[0] = r.obs[0]; ob[1] = r.obs[1]; ob[2] = r.obs[2];
      lvl = pts[i].anchor_level;
      if (gate_keep(r, R, T.v, cam, lvl)) {
        keep = 1;
        if (ob[0] > w0 * 0.5) ++right; else ++left;
        if (ob[1] > h0 * 0.5) ++lower; else ++upper;
      }
    }
    int s = keep;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, s, o); if ((threadIdx.x & 31) >= o) s += v; }
    if ((threadIdx.x & 31) == 31) sw[threadIdx.x >> 5] = s;
    __syncthreads();
    int before = 0;
    for (int k = 0; k < (int)(threadIdx.x >> 5); ++k) before += sw[k];
    const int at = carry + before + s - keep;
    if (keep) {
      track_point[at] = cpoint[i]; track_level[at] = lvl;
      track_uvu[3 * (size_t)at] = ob[0]; track_uvu[3 * (size_t)at + 1] = ob[1]; track_uvu[3 * (size_t)at + 2] = ob[2];
    }
    __syncthreads();
    if (threadIdx.x == kGate - 1) carry = at + keep;
    __syncthreads();
  }
  atomicAdd(&quad[0], left); atomicAdd(&quad[1], right); atomicAdd(&quad[2], upper); atomicAdd(&quad[3], lower);
  __syncthreads();
  if (threadIdx.x == 0) {
    ctl->n_tracks = carry;
    ctl->num_left = quad[0]; ctl->num_right = quad[1]; ctl->num_upper = quad[2]; ctl->num_lower = quad[3];
    // T_newloop_from_w = T_newloop_from_oldloop * T_query_from_loop^-1 * T_query_from_world (backend.cpp:964-966)
    double Tlq[7], A[7];
    svs::se3_inv(Tql.v, Tlq);
    svs::se3_mul(T.v, Tlq, A);
    svs::se3_mul(A, map_pose + 7 * (size_t)query, ctl->T_newloop_from_w);
  }
}


// ------------------------------------------------------------------ localRegisterFrame
// directNeighborsOf(root) (backend.cpp:433-449) and framesInNeighborhood(root, |direct| + 40) (slam_graph.cpp:105-140).
// As in graph.cu's k_bfs the queue discipline is the algorithm (a vertex joins when it is popped, the queue holds
// duplicates, a vertex outside the window is dropped when popped), so one thread walks it.  Only a vertex that joins
// pushes its neighbours, so the queue never holds more than 1 + nnzN entries.  direct[V], joined[V] and scan[V] come
// zeroed; scan = joined and not direct, the frames pointsVisibleInRoot reads.
__global__ void k_neighborhood(const int* __restrict__ nbr_ptr, const int* __restrict__ nbr_id, int root, const int* __restrict__ inwin,
                               int* __restrict__ direct, int* __restrict__ joined, int* __restrict__ scan, int* __restrict__ queue,
                               LoopCtl* ctl) {
  if (blockIdx.x || threadIdx.x) return;
  int nd = 1;
  direct[root] = 1;
  for (int i = nbr_ptr[root]; i < nbr_ptr[root + 1]; ++i)
    if (!direct[nbr_id[i]]) { direct[nbr_id[i]] = 1; ++nd; }
  const int size = nd + 40;   // NUM_FRAMES_TO_CHECK_FOR_REGISTRATION
  int head = 0, tail = 0, count = 0;
  queue[tail++] = root;
  while (head < tail && count < size) {
    const int v = queue[head++];
    if (joined[v] || !inwin[v]) continue;
    joined[v] = 1;
    scan[v] = !direct[v];
    ++count;
    for (int i = nbr_ptr[v]; i < nbr_ptr[v + 1]; ++i) queue[tail++] = nbr_id[i];   // strongest first
  }
  ctl->n_direct = nd;
  ctl->n_neighborhood = count;
}

// the vertices that anchor a candidate: the reference's vertex_table without root (pointsVisibleInRoot, :536-544)
__global__ void k_anchor_flag(int n, const int* __restrict__ anchor, const int* __restrict__ cpoint, int* __restrict__ anch) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) anch[anchor[cpoint[i]]] = 1;
}

// keyframesToRegister's reprojection test (backend.cpp:624-641) per match, with T_newroot_from_oldroot
__global__ void k_reg_gate(const svs_match_result* __restrict__ res, const svs_match_point* __restrict__ pts, int n, Pose7 T,
                           Cam4 cam, int* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double R[9];
  svs::quat_to_R(T.v, R);
  keep[i] = res[i].matched && gate_keep(res[i], R, T.v, cam, pts[i].anchor_level);
}

// a kept match becomes track gptr[i] (match order) and counts towards every vertex that observes its point, anchors a
// candidate and is not a direct neighbour (backend.cpp:643-691).  Integer atomics: the counts do not depend on the order
// the threads run in.  cnt[V][5] = strength, num_left, num_right, num_upper, num_lower under the reference's names,
// where u > w/2 counts as num_left.
__global__ void k_reg_count(svs::MapView m, const svs_match_result* __restrict__ res, const svs_match_point* __restrict__ pts,
                            const int* __restrict__ cpoint, int n, const int* __restrict__ keep, const int* __restrict__ gptr,
                            const int* __restrict__ anch, const int* __restrict__ direct, int w0, int h0, int* __restrict__ cnt,
                            int* __restrict__ track_point, double* __restrict__ track_uvu, int* __restrict__ track_level) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !keep[i]) return;
  const int at = gptr[i], p = cpoint[i];
  const double* ob = res[i].obs;
  track_point[at] = p;
  track_level[at] = pts[i].anchor_level;
  track_uvu[3 * (size_t)at] = ob[0]; track_uvu[3 * (size_t)at + 1] = ob[1]; track_uvu[3 * (size_t)at + 2] = ob[2];
  for (int k = m.vis_ptr[p]; k < m.vis_ptr[p + 1]; ++k) {
    const int v = m.vis_pose[k];
    if (!anch[v] || direct[v]) continue;
    int* c = cnt + 5 * (size_t)v;
    atomicAdd(c, 1);
    atomicAdd(c + (ob[0] > w0 * 0.5 ? 1 : 2), 1);
    atomicAdd(c + (ob[1] > h0 * 0.5 ? 4 : 3), 1);
  }
}

// the qualifying test of backend.cpp:697-704 per vertex; sflag = the vertex has an ImageStatsTable entry.  Vertex 0's
// thread also composes T_newroot_from_w = T_newroot_from_oldroot * T_root_from_world (:579-580).
__global__ void k_reg_qualify(int V, const int* __restrict__ cnt, int covis_thr, Pose7 T, const double* __restrict__ map_pose,
                              int root, int* __restrict__ sflag, int* __restrict__ qual, LoopCtl* ctl) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int* c = cnt + 5 * (size_t)v;
  const int half = covis_thr / 2;
  const int q = c[0] >= covis_thr && c[1] >= half && c[2] >= half && c[3] >= half && c[4] >= half;
  sflag[v] = c[0] > 0;
  qual[v] = q;
  if (q) atomicAdd(&ctl->n_neighbors, 1);
  if (v == 0) svs::se3_mul(T.v, map_pose + 7 * (size_t)root, ctl->T_newroot_from_w);
}

__global__ void k_reg_stats(int V, const int* __restrict__ cnt, const int* __restrict__ sflag, const int* __restrict__ sptr,
                            const int* __restrict__ qual, svs_register_stats* __restrict__ out) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V || !sflag[v]) return;
  const int* c = cnt + 5 * (size_t)v;
  svs_register_stats s;
  s.vertex = v;
  s.strength = c[0]; s.num_left = c[1]; s.num_right = c[2]; s.num_upper = c[3]; s.num_lower = c[4];
  s.qualified = qual[v];
  out[sptr[v]] = s;
}

// registerKeyframes' trackpoint_list (backend.cpp:702-712): a track is committed when a qualifying vertex observes its
// point.  The reference lists such a point once per qualifying vertex, with the same feature each time, and
// feature_table.insert keeps the first: committing each track once is the same map.
__global__ void k_reg_commit_flag(svs::MapView m, int nt, const int* __restrict__ track_point, const int* __restrict__ qual,
                                  int* __restrict__ flag) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  const int p = track_point[t];
  int f = 0;
  for (int k = m.vis_ptr[p]; k < m.vis_ptr[p + 1]; ++k) f |= qual[m.vis_pose[k]];
  flag[t] = f;
}

__global__ void k_reg_commit_emit(int nt, const int* __restrict__ flag, const int* __restrict__ ptr, const int* __restrict__ tp,
                                  const double* __restrict__ tu, const int* __restrict__ tl, int* __restrict__ op,
                                  double* __restrict__ ou, int* __restrict__ ol) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt || !flag[t]) return;
  const int at = ptr[t];
  op[at] = tp[t]; ol[at] = tl[t];
  for (int k = 0; k < 3; ++k) ou[3 * (size_t)at + k] = tu[3 * (size_t)t + k];
}

// ------------------------------------------------------------------ host steps shared by both entry points

struct CandBufs {
  int *flag, *qptr, *qpts, *cflag, *cptr, *cpt;   // [Np], [Np+1], [Np], [Np], [Np+1], [Np]
  svs_match_point *rec, *pts;                     // [Np], [Np]
};

// the per-call buffers of both entry points (Nq = max(Np, 1)): the control block, the window's flags, the vertices'
// slots, the candidate scan, the matcher's slot poses saved for a refusal, and the gated tracks
struct LoopBufs {
  LoopCtl* ctl; int *win, *slot; CandBufs cb; double* save;
  int* tp; double* tu; int* tl;   // [Nq], [Nq][3], [Nq]
};
LoopBufs loop_carve(svs::Bump& m, int V, int Nq, int max_kf) {
  LoopBufs b;
  b.ctl = m.take<LoopCtl>(1); b.win = m.take<int>(V); b.slot = m.take<int>(V);
  b.cb.flag = m.take<int>(Nq); b.cb.qptr = m.take<int>(Nq + 1); b.cb.qpts = m.take<int>(Nq);
  b.cb.cflag = m.take<int>(Nq); b.cb.cptr = m.take<int>(Nq + 1);
  b.cb.rec = m.take<svs_match_point>(Nq); b.cb.pts = m.take<svs_match_point>(Nq); b.cb.cpt = m.take<int>(Nq);
  b.save = m.take<double>(7 * (size_t)max_kf);
  b.tp = m.take<int>(Nq); b.tu = m.take<double>(3 * (size_t)Nq); b.tl = m.take<int>(Nq);
  return b;
}

// what svs_localRegisterFrame takes after loop_carve; dir .. cnt are zeroed together (zero_bytes from dir on)
struct RegBufs {
  int *dir, *join, *scan, *anch, *cnt;   // [V] x 4, [5][V]
  size_t zero_bytes;
  int *sflag, *sptr, *qual, *queue, *keep, *gptr, *mflag, *mptr, *mp, *ml; double* mu; svs_register_stats* stats;
};
RegBufs reg_carve(svs::Bump& m, int V, int Nq, int nnzN) {
  RegBufs r;
  const size_t z = m.off;
  r.dir = m.take<int>(V); r.join = m.take<int>(V); r.scan = m.take<int>(V); r.anch = m.take<int>(V);
  r.cnt = m.take<int>(5 * (size_t)V);
  r.zero_bytes = m.off - z;
  r.sflag = m.take<int>(V); r.sptr = m.take<int>(V + 1); r.qual = m.take<int>(V);
  r.stats = m.take<svs_register_stats>(V); r.queue = m.take<int>((size_t)nnzN + 1);
  r.keep = m.take<int>(Nq); r.gptr = m.take<int>(Nq + 1);
  r.mflag = m.take<int>(Nq); r.mptr = m.take<int>(Nq + 1);
  r.mp = m.take<int>(Nq); r.mu = m.take<double>(3 * (size_t)Nq); r.ml = m.take<int>(Nq);
  return r;
}

// the candidate scan: the points some vertex of vset[V] observes, in ascending index, then those anchored in the window
// whose (int) projection from T_ref_from_w (device memory) lies in the anchor level's image (k_cand_test).  Waits for
// the stream; *nc = the number of candidates, compacted into b.pts / b.cpt.
cudaError_t scan_candidates(const svs::MapView& m, const int* vset, const int* inwin, const int* slot, const Levels& lv,
                            const double* T_ref_from_w, LoopCtl* ctl, const CandBufs& b, cudaStream_t st, int* nc) {
  const int Np = m.Np;
  int nq = 0;
  *nc = 0;
  if (!Np) return cudaStreamSynchronize(st);
  const int bP = (Np + 255) / 256;
  k_query_flag<<<bP, 256, 0, st>>>(m, vset, b.flag);
  svs::launch_scan(b.flag, Np, b.qptr, st);
  k_compact_ids<<<bP, 256, 0, st>>>(Np, b.flag, b.qptr, b.qpts);
  cudaError_t e = cudaMemcpyAsync(&nq, b.qptr + Np, sizeof(int), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess || !nq) return e;
  const int bq = (nq + 255) / 256;
  k_cand_test<<<bq, 256, 0, st>>>(m, b.qpts, b.qptr, inwin, slot, lv, T_ref_from_w, ctl, b.cflag, b.rec);
  svs::launch_scan(b.cflag, nq, b.cptr, st);
  k_cand_emit<<<bq, 256, 0, st>>>(Np, b.qptr, b.qpts, b.cflag, b.cptr, b.rec, b.pts, b.cpt);
  e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpyAsync(nc, b.cptr + nq, sizeof(int), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  return e;
}

// the findings of the candidate scan that refuse the call, nullptr when there are none
const char* candidate_refusal(const LoopCtl& c, int nc, const svs::MatcherView& mv, int max_obs) {
  if (c.no_anchor_obs) return "a candidate's anchor frame has no observation of it";
  if (c.bad_level) return "a candidate's anchor level is not a level of the matcher";
  if (c.no_slot) return "a candidate's anchor frame has no matcher slot";
  if (nc > mv.max_pts || nc > max_obs) return "more candidates than the matcher's max_points or the pose handle's max_obs";
  return nullptr;
}

void launch_slot_copy(const svs::MatcherView& mv, double* save, int dir, cudaStream_t st) {
  k_slot_copy<<<(7 * mv.max_kf + 255) / 256, 256, 0, st>>>(mv.max_kf, mv.slot_T, mv.slot_stride, save, dir);
}

// matchAndAlign (backend.cpp:725-784) on the nc candidates d_pts: svs_match at radius 10 with T_cur_from_actkey = I, the
// LM (true, 2, 25) -> T_align1, svs_match at radius 4 from there, the LM (true, 2, 15) -> T.  *first_short = 1 when the
// first match found fewer than covis_thr (nothing after it ran); the second round's count is left to the caller.
// Returns SVS_OK or the matcher's / LM's error (message in *cerr; SVS_ERR_NUMERIC for a NaN residual).
int match_and_align(svs_matcher* mt, svs_pose* po, const svs_cam* cam, const double T_actkey_from_w[7],
                    const svs_match_point* d_pts, int nc, int covis_thr, LoopCtl* d_ctl, cudaStream_t st, int nm[2],
                    double T_align1[7], double T[7], svs_pose_stats lm[2], const svs_match_result** d_res, int* first_short,
                    std::string* cerr) {
  const double I7[7] = {0, 0, 0, 1, 0, 0, 0};
  const svs_pose_params p25 = {1, 2.0, 25, -1.0, 0.00001}, p15 = {1, 2.0, 15, -1.0, 0.00001};
  int nres = 0, rdev = 0;
  *first_short = 0;
  memcpy(T, I7, sizeof I7);
  for (int round = 0; round < 2; ++round) {
    int rc = svs::match_device(mt, T, T_actkey_from_w, d_pts, nc, round == 0 ? 10 : 4, 22, 10);
    if (rc != SVS_OK) { *cerr = std::string("svs_match: ") + svs_matcher_last_error(mt); return rc; }
    svs::matcher_device_results(mt, d_res, &nres, &rdev);
    nm[round] = 0;
    if (nc) {
      k_count_matched<<<1, kGate, 0, st>>>(*d_res, nc, d_ctl);
      cudaError_t e = cudaGetLastError();
      if (e == cudaSuccess) e = cudaMemcpyAsync(&nm[round], &d_ctl->n_matched, sizeof(int), cudaMemcpyDeviceToHost, st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
      if (e != cudaSuccess) { *cerr = std::string("matchAndAlign: ") + cudaGetErrorString(e); return SVS_ERR_CUDA; }
    }
    if (round == 0 && nm[0] < covis_thr) { *first_short = 1; return SVS_OK; }
    rc = svs_calcFastMotionOnly_matched(po, mt, cam, round == 0 ? &p25 : &p15, T, &lm[round]);
    if (rc != SVS_OK) { *cerr = std::string("calcFastMotionOnly: ") + svs_pose_last_error(po); return rc; }
    if (round == 0) memcpy(T_align1, T, sizeof I7);
  }
  return SVS_OK;
}

Levels matcher_levels(const svs::MatcherView& mv) {
  Levels lv{};
  lv.n = mv.nlevels;
  for (int l = 0; l < mv.nlevels; ++l) { lv.w[l] = mv.lv[l].w; lv.h[l] = mv.lv[l].h; lv.f[l] = mv.lv[l].f; lv.px[l] = mv.lv[l].px; lv.py[l] = mv.lv[l].py; }
  return lv;
}

// the refusals both entry points share: a window vertex listed twice or outside [0, V), a slot outside the matcher or
// used twice; inwin[V] receives the window's flags
const char* window_and_slot_refusal(int V, int P, const int* window_vertex, const int* vertex_slot, int max_kf,
                                    std::vector<int>& inwin) {
  std::vector<int> used(max_kf, 0);
  inwin.assign(V, 0);
  for (int i = 0; i < P; ++i) {
    const int v = window_vertex[i];
    if (v < 0 || v >= V || inwin[v]) return "window names a vertex twice or outside [0, V)";
    inwin[v] = 1;
  }
  for (int v = 0; v < V; ++v) {
    const int s = vertex_slot[v];
    if (s < -1 || s >= max_kf || (s >= 0 && used[s]++)) return "vertex_slot names a slot outside the matcher or twice";
  }
  return nullptr;
}

}  // namespace

#define LCK(call)                                                                   \
  do {                                                                              \
    cudaError_t e_ = (call);                                                        \
    if (e_ != cudaSuccess) { cerr = std::string(#call) + ": " + cudaGetErrorString(e_); rc = SVS_ERR_CUDA; goto done; } \
  } while (0)

extern "C" int svs_globalLoopClosure(svs_map* map, svs_matcher* mt, svs_pose* po, const svs_cam* cam, int covis_thr, int query,
                                     int loop, const double T_query_from_loop[7], int P, const int* window_vertex,
                                     const int* vertex_slot, svs_loop_result* res, int cap, int* track_point, double* track_uvu,
                                     int* track_level) {
  svs::NvtxRange nvtx_("globalLoopClosure");
  if (!map) return SVS_ERR_INVALID;
  svs::MapView m;
  svs::map_view(map, &m);
  auto refuse = [&](const char* msg) { return svs::fail(m.base, SVS_ERR_INVALID, msg); };
  if (!mt || !po || !cam || !T_query_from_loop || !res || !vertex_slot || P < 0 || (P && !window_vertex) || cap < 0 ||
      (cap && (!track_point || !track_uvu || !track_level)))
    return refuse("svs_globalLoopClosure: null argument or negative size");
  memset(res, 0, sizeof *res);
  svs::MatcherView mv;
  svs::matcher_view(mt, &mv);
  int pdev = -1, max_obs = 0;
  svs::pose_capacity(po, &pdev, &max_obs);
  const int V = m.V, Np = m.Np;
  if (V <= 0) return refuse("svs_globalLoopClosure: the map is empty");
  if (query < 0 || query >= V || loop < 0 || loop >= V || query == loop) return refuse("query or loop outside [0, V), or query == loop");
  if (covis_thr < 1) return refuse("covis_thr < 1");
  if (mv.device != m.device || pdev != m.device) return refuse("map, matcher and pose handle live on different devices");
  std::vector<int> inwin;
  if (const char* why = window_and_slot_refusal(V, P, window_vertex, vertex_slot, mv.max_kf, inwin)) return refuse(why);
  std::vector<int> qset(V, 0);
  qset[query] = 1;
  cudaSetDevice(m.device);
  cudaStream_t st = m.stream;
  const int Nq = std::max(Np, 1);
  svs::Bump m0{nullptr};
  loop_carve(m0, V, Nq, mv.max_kf);
  m0.take<int>(V);   // qset
  char* W = nullptr;
  std::string cerr;
  int rc = SVS_OK;
  bool refreshed = false;
  LoopCtl c{};
  Pose7 Tql;
  memcpy(Tql.v, T_query_from_loop, sizeof Tql.v);
  LoopBufs b{};
  int* d_qset = nullptr;
  {
    LCK(cudaStreamSynchronize(st));
    LCK(cudaMalloc(&W, m0.off));
    svs::Bump mw{W};
    b = loop_carve(mw, V, Nq, mv.max_kf);
    d_qset = mw.take<int>(V);
    LCK(cudaMemsetAsync(b.ctl, 0, sizeof(LoopCtl), st));
    LCK(cudaMemcpyAsync(b.win, inwin.data(), sizeof(int) * V, cudaMemcpyHostToDevice, st));
    LCK(cudaMemcpyAsync(b.slot, vertex_slot, sizeof(int) * V, cudaMemcpyHostToDevice, st));
    LCK(cudaMemcpyAsync(d_qset, qset.data(), sizeof(int) * V, cudaMemcpyHostToDevice, st));
    // 1 candidates
    k_loop_setup<<<1, 32, 0, st>>>(m.pose, query, Tql, b.ctl);
    int nc = 0;
    LCK(scan_candidates(m, d_qset, b.win, b.slot, matcher_levels(mv), b.ctl->T_loop_from_w, b.ctl, b.cb, st, &nc));
    LCK(cudaGetLastError());
    LCK(cudaMemcpyAsync(&c, b.ctl, sizeof c, cudaMemcpyDeviceToHost, st));
    LCK(cudaStreamSynchronize(st));
    res->n_candidates = nc;
    if (const char* why = candidate_refusal(c, nc, mv, max_obs)) { cerr = why; rc = SVS_ERR_INVALID; goto done; }
    launch_slot_copy(mv, b.save, 0, st);
    k_slot_refresh<<<(7 * V + 255) / 256, 256, 0, st>>>(V, m.pose, b.slot, loop, b.ctl->T_loop_from_w, mv.slot_T, mv.slot_stride);
    LCK(cudaGetLastError());
    LCK(cudaStreamSynchronize(st));   // the matcher's stream reads the slots and the candidates
    refreshed = true;
    // 2 matchAndAlign
    const svs_match_result* d_res = nullptr;
    double T[7];
    int nm[2] = {0, 0}, first_short = 0;
    rc = match_and_align(mt, po, cam, c.T_loop_from_w, b.cb.pts, nc, covis_thr, b.ctl, st, nm, res->T_align1, T, res->lm, &d_res,
                         &first_short, &cerr);
    res->n_matched1 = nm[0];
    if (rc != SVS_OK) goto done;
    if (first_short) { res->stage = 1; goto done; }
    res->n_matched2 = nm[1];
    memcpy(res->T_newloop_from_oldloop, T, sizeof T);
    if (res->n_matched2 < covis_thr) { res->stage = 2; goto done; }
    // 3 gate
    Pose7 Tn;
    memcpy(Tn.v, T, sizeof T);
    const Cam4 c4{cam->f, cam->px, cam->py, cam->b};
    k_gate<<<1, kGate, 0, st>>>(d_res, b.cb.pts, b.cb.cpt, nc, Tn, Tql, c4, mv.lv[0].w, mv.lv[0].h, m.pose, query, b.ctl, b.tp,
                                b.tu, b.tl);
    LCK(cudaGetLastError());
    LCK(cudaMemcpyAsync(&c, b.ctl, sizeof c, cudaMemcpyDeviceToHost, st));
    LCK(cudaStreamSynchronize(st));
    const int nt = c.n_tracks;
    res->n_tracks = nt;
    res->num_left = c.num_left; res->num_right = c.num_right; res->num_upper = c.num_upper; res->num_lower = c.num_lower;
    if (nt > cap) { cerr = "cap is smaller than the number of tracks"; rc = SVS_ERR_INVALID; goto done; }
    if (nt) {
      LCK(cudaMemcpyAsync(track_point, b.tp, sizeof(int) * nt, cudaMemcpyDeviceToHost, st));
      LCK(cudaMemcpyAsync(track_uvu, b.tu, sizeof(double) * 3 * nt, cudaMemcpyDeviceToHost, st));
      LCK(cudaMemcpyAsync(track_level, b.tl, sizeof(int) * nt, cudaMemcpyDeviceToHost, st));
      LCK(cudaStreamSynchronize(st));
    }
    const int half = covis_thr / 2;
    if (nt < covis_thr) { res->stage = 3; goto done; }
    if (c.num_lower < half || c.num_upper < half || c.num_left < half || c.num_right < half) { res->stage = 4; goto done; }
    // 4 commit
    memcpy(res->T_newloop_from_w, c.T_newloop_from_w, sizeof c.T_newloop_from_w);
    rc = svs::map_add_observations(map, loop, nt, b.tp, b.tu, b.tl);
    if (rc != SVS_OK) { cerr = svs_map_last_error(map); goto done; }
    res->verified = 1;
    res->stage = 0;
  }
done:
  if (rc != SVS_OK && refreshed && rc != SVS_ERR_NUMERIC) {   // a refusal leaves the slots as they were
    launch_slot_copy(mv, b.save, 1, st);
    cudaStreamSynchronize(st);
  }
  if (W) { cudaStreamSynchronize(st); cudaFree(W); }
  if (rc != SVS_OK) m.base->err = cerr;
  return rc;
}

extern "C" int svs_localRegisterFrame(svs_map* map, svs_matcher* mt, svs_pose* po, const svs_cam* cam, int covis_thr, int root,
                                      int P, const int* window_vertex, const int* vertex_slot, svs_register_result* res,
                                      int cap_stats, svs_register_stats* stats, int cap_tracks, int* track_point,
                                      double* track_uvu, int* track_level, int* track_committed) {
  svs::NvtxRange nvtx_("localRegisterFrame");
  if (!map) return SVS_ERR_INVALID;
  svs::MapView m;
  svs::map_view(map, &m);
  auto refuse = [&](const char* msg) { return svs::fail(m.base, SVS_ERR_INVALID, msg); };
  if (!mt || !po || !cam || !res || !vertex_slot || P < 0 || (P && !window_vertex) || cap_stats < 0 || cap_tracks < 0 ||
      (cap_stats && !stats) || (cap_tracks && (!track_point || !track_uvu || !track_level || !track_committed)))
    return refuse("svs_localRegisterFrame: null argument or negative size");
  memset(res, 0, sizeof *res);
  const int* nbr_ptr = nullptr;
  const int* nbr_id = nullptr;
  int nnzN = 0;
  if (!svs::map_graph(map, &nbr_ptr, &nbr_id, &nnzN))
    return svs::fail(m.base, SVS_ERR_STATE, "svs_map_set_graph has not been called for this map");
  svs::MatcherView mv;
  svs::matcher_view(mt, &mv);
  int pdev = -1, max_obs = 0;
  svs::pose_capacity(po, &pdev, &max_obs);
  const int V = m.V, Np = m.Np;
  if (V <= 0) return refuse("svs_localRegisterFrame: the map is empty");
  if (root < 0 || root >= V) return refuse("root outside [0, V)");
  if (covis_thr < 1) return refuse("covis_thr < 1");
  if (mv.device != m.device || pdev != m.device) return refuse("map, matcher and pose handle live on different devices");
  std::vector<int> inwin;
  if (const char* why = window_and_slot_refusal(V, P, window_vertex, vertex_slot, mv.max_kf, inwin)) return refuse(why);
  cudaSetDevice(m.device);
  cudaStream_t st = m.stream;
  const int Nq = std::max(Np, 1);
  svs::Bump m0{nullptr};
  loop_carve(m0, V, Nq, mv.max_kf);
  reg_carve(m0, V, Nq, nnzN);
  char* W = nullptr;
  std::string cerr;
  int rc = SVS_OK;
  bool refreshed = false;
  LoopCtl c{};
  LoopBufs b{};
  RegBufs r{};
  {
    LCK(cudaStreamSynchronize(st));
    LCK(cudaMalloc(&W, m0.off));
    svs::Bump mw{W};
    b = loop_carve(mw, V, Nq, mv.max_kf);
    r = reg_carve(mw, V, Nq, nnzN);
    LCK(cudaMemsetAsync(b.ctl, 0, sizeof(LoopCtl), st));
    LCK(cudaMemsetAsync(r.dir, 0, r.zero_bytes, st));
    LCK(cudaMemcpyAsync(b.win, inwin.data(), sizeof(int) * V, cudaMemcpyHostToDevice, st));
    LCK(cudaMemcpyAsync(b.slot, vertex_slot, sizeof(int) * V, cudaMemcpyHostToDevice, st));
    // 1 neighbourhoods and candidates (pointsVisibleInRoot, backend.cpp:472-546)
    k_neighborhood<<<1, 32, 0, st>>>(nbr_ptr, nbr_id, root, b.win, r.dir, r.join, r.scan, r.queue, b.ctl);
    const double* d_Troot = m.pose + 7 * (size_t)root;
    int nc = 0;
    LCK(scan_candidates(m, r.scan, b.win, b.slot, matcher_levels(mv), d_Troot, b.ctl, b.cb, st, &nc));
    if (nc) k_anchor_flag<<<(nc + 255) / 256, 256, 0, st>>>(nc, m.anchor, b.cb.cpt, r.anch);
    LCK(cudaGetLastError());
    LCK(cudaMemcpyAsync(&c, b.ctl, sizeof c, cudaMemcpyDeviceToHost, st));
    double Troot[7];
    LCK(cudaMemcpyAsync(Troot, d_Troot, sizeof Troot, cudaMemcpyDeviceToHost, st));
    LCK(cudaStreamSynchronize(st));
    res->n_direct = c.n_direct;
    res->n_neighborhood = c.n_neighborhood;
    res->n_candidates = nc;
    if (const char* why = candidate_refusal(c, nc, mv, max_obs)) { cerr = why; rc = SVS_ERR_INVALID; goto done; }
    if (nc < covis_thr) { res->stage = 1; goto done; }
    launch_slot_copy(mv, b.save, 0, st);
    k_slot_refresh<<<(7 * V + 255) / 256, 256, 0, st>>>(V, m.pose, b.slot, -1, nullptr, mv.slot_T, mv.slot_stride);
    LCK(cudaGetLastError());
    LCK(cudaStreamSynchronize(st));   // the matcher's stream reads the slots and the candidates
    refreshed = true;
    // 2 matchAndAlign
    const svs_match_result* d_res = nullptr;
    double T[7];
    int nm[2] = {0, 0}, first_short = 0;
    rc = match_and_align(mt, po, cam, Troot, b.cb.pts, nc, covis_thr, b.ctl, st, nm, res->T_align1, T, res->lm, &d_res,
                         &first_short, &cerr);
    res->n_matched1 = nm[0];
    if (rc != SVS_OK) goto done;
    if (first_short) { res->stage = 2; goto done; }
    res->n_matched2 = nm[1];
    memcpy(res->T_newroot_from_oldroot, T, sizeof T);
    if (res->n_matched2 < covis_thr) { res->stage = 3; goto done; }
    // 3 keyframesToRegister (backend.cpp:615-722)
    Pose7 Tn;
    memcpy(Tn.v, T, sizeof T);
    const Cam4 c4{cam->f, cam->px, cam->py, cam->b};
    const int bc = (nc + 255) / 256, bV = (V + 255) / 256;
    k_reg_gate<<<bc, 256, 0, st>>>(d_res, b.cb.pts, nc, Tn, c4, r.keep);
    svs::launch_scan(r.keep, nc, r.gptr, st);
    k_reg_count<<<bc, 256, 0, st>>>(m, d_res, b.cb.pts, b.cb.cpt, nc, r.keep, r.gptr, r.anch, r.dir, mv.lv[0].w,
                                     mv.lv[0].h, r.cnt, b.tp, b.tu, b.tl);
    k_reg_qualify<<<bV, 256, 0, st>>>(V, r.cnt, covis_thr, Tn, m.pose, root, r.sflag, r.qual, b.ctl);
    svs::launch_scan(r.sflag, V, r.sptr, st);
    k_reg_stats<<<bV, 256, 0, st>>>(V, r.cnt, r.sflag, r.sptr, r.qual, r.stats);
    LCK(cudaGetLastError());
    int nt = 0, ns = 0;
    LCK(cudaMemcpyAsync(&nt, r.gptr + nc, sizeof(int), cudaMemcpyDeviceToHost, st));
    LCK(cudaMemcpyAsync(&ns, r.sptr + V, sizeof(int), cudaMemcpyDeviceToHost, st));
    LCK(cudaMemcpyAsync(&c, b.ctl, sizeof c, cudaMemcpyDeviceToHost, st));
    LCK(cudaStreamSynchronize(st));
    res->n_tracks = nt;
    res->n_stats = ns;
    res->n_neighbors = c.n_neighbors;
    if (nt > cap_tracks || ns > cap_stats) { cerr = "cap_tracks or cap_stats is smaller than the tracks or the stats table"; rc = SVS_ERR_INVALID; goto done; }
    int ncommit = 0;
    if (nt) {
      const int bt = (nt + 255) / 256;
      k_reg_commit_flag<<<bt, 256, 0, st>>>(m, nt, b.tp, r.qual, r.mflag);
      svs::launch_scan(r.mflag, nt, r.mptr, st);
      k_reg_commit_emit<<<bt, 256, 0, st>>>(nt, r.mflag, r.mptr, b.tp, b.tu, b.tl,
                                            r.mp, r.mu, r.ml);
      LCK(cudaGetLastError());
      LCK(cudaMemcpyAsync(&ncommit, r.mptr + nt, sizeof(int), cudaMemcpyDeviceToHost, st));
      LCK(cudaMemcpyAsync(track_point, b.tp, sizeof(int) * nt, cudaMemcpyDeviceToHost, st));
      LCK(cudaMemcpyAsync(track_uvu, b.tu, sizeof(double) * 3 * nt, cudaMemcpyDeviceToHost, st));
      LCK(cudaMemcpyAsync(track_level, b.tl, sizeof(int) * nt, cudaMemcpyDeviceToHost, st));
      LCK(cudaMemcpyAsync(track_committed, r.mflag, sizeof(int) * nt, cudaMemcpyDeviceToHost, st));
    }
    if (ns) LCK(cudaMemcpyAsync(stats, r.stats, sizeof(svs_register_stats) * ns, cudaMemcpyDeviceToHost, st));
    LCK(cudaStreamSynchronize(st));
    if (c.n_neighbors == 0) { res->stage = 4; goto done; }
    // 4 commit (registerKeyframes' addNewObsToOldPoints, slam_graph.cpp:189-205); root's pose stays
    res->n_committed = ncommit;
    memcpy(res->T_newroot_from_w, c.T_newroot_from_w, sizeof c.T_newroot_from_w);
    rc = svs::map_add_observations(map, root, ncommit, r.mp, r.mu, r.ml);
    if (rc != SVS_OK) { cerr = svs_map_last_error(map); goto done; }
    res->registered = 1;
    res->stage = 0;
  }
done:
  if (rc != SVS_OK && refreshed && rc != SVS_ERR_NUMERIC) {   // a refusal leaves the slots as they were
    launch_slot_copy(mv, b.save, 1, st);
    cudaStreamSynchronize(st);
  }
  if (W) { cudaStreamSynchronize(st); cudaFree(W); }
  if (rc != SVS_OK) m.base->err = cerr;
  return rc;
}
#undef LCK
