// loop.cu -- metric verification of a proposed loop on sm_90a: Backend::globalLoopClosure (scavislam/backend.cpp:830-1001)
// with matchAndAlign (:726-784) from the device map, the matcher's keyframe slots and the motion-only LM, and the
// commit of SlamGraph::addLoopClosure's addNewObsToOldPoints on the loop vertex (slam_graph.cpp:220, 400-420).
//
// Kernels of this file: the candidate scan (points the query observes: flag / scan / compact over the map, then test /
// scan / emit over those), the slot-pose refresh and the one-CTA gate.  Matching, the LM and the observation commit
// run in match.cu, pose.cu and graph.cu.  The projections are compiled with -fmad=false and written operation by
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

__global__ void k_query_flag(svs::MapView m, int query, int* __restrict__ flag) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= m.Np) return;
  int f = 0;
  for (int i = m.vis_ptr[p]; i < m.vis_ptr[p + 1]; ++i) f |= m.vis_pose[i] == query;
  flag[p] = f;
}

__global__ void k_compact_ids(int n, const int* __restrict__ flag, const int* __restrict__ ptr, int* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flag[i]) out[ptr[i]] = i;
}

// the candidate test of backend.cpp:853-893 for the nq points the query observes (qpts, ascending)
__global__ void k_cand_test(svs::MapView m, const int* __restrict__ qpts, const int* __restrict__ qptr, const int* __restrict__ inwin,
                            const int* __restrict__ slot, Levels lv, LoopCtl* ctl, int* __restrict__ cflag,
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
  svs::se3_mul(ctl->T_loop_from_w, Twa, Tla);
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

// the reference's vertex_table: every slot gets its vertex's map pose, loop's slot the predicted T_loop_from_world.
// Only the device copy of the slot poses changes; the matcher's host mirror keeps the poses last set through the C ABI.
// That is safe as long as the matcher uploads a slot's record only right after setting that slot's pose
// (svs_matcher_set_keyframe, svs_matcher_set_pyramid_device), which is how match.cu does it.
__global__ void k_slot_refresh(int V, const double* __restrict__ map_pose, const int* __restrict__ slot, int loop, const LoopCtl* ctl,
                               double* __restrict__ slot_T, size_t stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 7 * V) return;
  const int v = i / 7, q = i % 7;
  if (slot[v] < 0) return;
  double* t = reinterpret_cast<double*>(reinterpret_cast<char*>(slot_T) + (size_t)slot[v] * stride);
  t[q] = v == loop ? ctl->T_loop_from_w[q] : map_pose[7 * (size_t)v + q];
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
  const double t0 = T.v[4], t1 = T.v[5], t2 = T.v[6];
  int left = 0, right = 0, upper = 0, lower = 0;
  __syncthreads();
  for (int base = 0; base < n; base += kGate) {
    const int i = base + threadIdx.x;
    int keep = 0;
    double ob[3] = {0, 0, 0};
    int lvl = 0;
    if (i < n && res[i].matched) {
      const svs_match_result& r = res[i];
      const double X0 = r.xyz_actkey[0], X1 = r.xyz_actkey[1], X2 = r.xyz_actkey[2];
      const double x = R[0] * X0 + R[1] * X1 + R[2] * X2 + t0;
      const double y = R[3] * X0 + R[4] * X1 + R[5] * X2 + t1;
      const double z = R[6] * X0 + R[7] * X1 + R[8] * X2 + t2;
      ob[0] = r.obs[0]; ob[1] = r.obs[1]; ob[2] = r.obs[2];
      const double d0 = ob[0] - (cam.f * (x / z) + cam.px);
      const double d1 = ob[1] - (cam.f * (y / z) + cam.py);
      const double d2 = ob[2] - ((x - cam.b) / z * cam.f + cam.px);
      lvl = pts[i].anchor_level;
      const int factor = 1 << lvl;   // zeroFromPyr_i(1, level)
      if (fabs(d0) < 2.0 * factor && fabs(d1) < 2.0 * factor && fabs(d2) < 2.0 * 3) {
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

size_t al256(size_t x) { return (x + 255) / 256 * 256; }

}  // namespace

extern "C" int svs_globalLoopClosure(svs_map* map, svs_matcher* mt, svs_pose* po, const svs_cam* cam, int covis_thr, int query,
                                     int loop, const double T_query_from_loop[7], int P, const int* window_vertex,
                                     const int* vertex_slot, svs_loop_result* res, int cap, int* track_point, double* track_uvu,
                                     int* track_level) {
  svs::NvtxRange nvtx_("globalLoopClosure");
  if (!map) return SVS_ERR_INVALID;
  auto refuse = [&](const char* msg) { svs::map_set_error(map, msg); return SVS_ERR_INVALID; };
  if (!mt || !po || !cam || !T_query_from_loop || !res || !vertex_slot || P < 0 || (P && !window_vertex) || cap < 0 ||
      (cap && (!track_point || !track_uvu || !track_level)))
    return refuse("svs_globalLoopClosure: null argument or negative size");
  memset(res, 0, sizeof *res);
  svs::MapView m;
  svs::map_view(map, &m);
  svs::MatcherView mv;
  svs::matcher_view(mt, &mv);
  int pdev = -1, max_obs = 0;
  svs::pose_capacity(po, &pdev, &max_obs);
  const int V = m.V, Np = m.Np;
  if (V <= 0) return refuse("svs_globalLoopClosure: the map is empty");
  if (query < 0 || query >= V || loop < 0 || loop >= V || query == loop) return refuse("query or loop outside [0, V), or query == loop");
  if (covis_thr < 1) return refuse("covis_thr < 1");
  if (mv.device != m.device || pdev != m.device) return refuse("map, matcher and pose handle live on different devices");
  std::vector<int> inwin(V, 0), used(mv.max_kf, 0);
  for (int i = 0; i < P; ++i) {
    const int v = window_vertex[i];
    if (v < 0 || v >= V || inwin[v]) return refuse("window names a vertex twice or outside [0, V)");
    inwin[v] = 1;
  }
  for (int v = 0; v < V; ++v) {
    const int s = vertex_slot[v];
    if (s < -1 || s >= mv.max_kf || (s >= 0 && used[s]++)) return refuse("vertex_slot names a slot outside the matcher or twice");
  }
  cudaSetDevice(m.device);
  cudaStream_t st = m.stream;
  const int Nq = std::max(Np, 1);
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += al256(bytes); return o; };
  const size_t o_ctl = take(sizeof(LoopCtl)), o_win = take(sizeof(int) * V), o_slot = take(sizeof(int) * V);
  const size_t o_flag = take(sizeof(int) * Nq), o_qptr = take(sizeof(int) * (Nq + 1)), o_qpts = take(sizeof(int) * Nq);
  const size_t o_cflag = take(sizeof(int) * Nq), o_cptr = take(sizeof(int) * (Nq + 1));
  const size_t o_rec = take(sizeof(svs_match_point) * Nq), o_pts = take(sizeof(svs_match_point) * Nq);
  const size_t o_cpt = take(sizeof(int) * Nq), o_save = take(sizeof(double) * 7 * mv.max_kf);
  const size_t o_tp = take(sizeof(int) * Nq), o_tu = take(sizeof(double) * 3 * Nq), o_tl = take(sizeof(int) * Nq);
  char* W = nullptr;
  std::string cerr;
  int rc = SVS_OK;
  bool refreshed = false;
  LoopCtl c{};
  Pose7 Tql;
  memcpy(Tql.v, T_query_from_loop, sizeof Tql.v);
  auto I = [&](size_t o) { return reinterpret_cast<int*>(W + o); };
  LoopCtl* d_ctl = reinterpret_cast<LoopCtl*>(W + o_ctl);
  svs_match_point* d_pts = nullptr;
#define LCK(call)                                                                   \
  do {                                                                              \
    cudaError_t e_ = (call);                                                        \
    if (e_ != cudaSuccess) { cerr = std::string(#call) + ": " + cudaGetErrorString(e_); rc = SVS_ERR_CUDA; goto done; } \
  } while (0)
  {
    LCK(cudaStreamSynchronize(st));
    LCK(cudaMalloc(&W, off));
    d_ctl = reinterpret_cast<LoopCtl*>(W + o_ctl);
    d_pts = reinterpret_cast<svs_match_point*>(W + o_pts);
    LCK(cudaMemsetAsync(d_ctl, 0, sizeof(LoopCtl), st));
    LCK(cudaMemcpyAsync(I(o_win), inwin.data(), sizeof(int) * V, cudaMemcpyHostToDevice, st));
    LCK(cudaMemcpyAsync(I(o_slot), vertex_slot, sizeof(int) * V, cudaMemcpyHostToDevice, st));
    Levels lv{};
    lv.n = mv.nlevels;
    for (int l = 0; l < mv.nlevels; ++l) { lv.w[l] = mv.lv[l].w; lv.h[l] = mv.lv[l].h; lv.f[l] = mv.lv[l].f; lv.px[l] = mv.lv[l].px; lv.py[l] = mv.lv[l].py; }
    // 1 candidates
    k_loop_setup<<<1, 32, 0, st>>>(m.pose, query, Tql, d_ctl);
    int nq = 0, nc = 0;
    if (Np) {
      const int bP = (Np + 255) / 256;
      k_query_flag<<<bP, 256, 0, st>>>(m, query, I(o_flag));
      svs::launch_scan(I(o_flag), Np, I(o_qptr), st);
      k_compact_ids<<<bP, 256, 0, st>>>(Np, I(o_flag), I(o_qptr), I(o_qpts));
      LCK(cudaMemcpyAsync(&nq, I(o_qptr) + Np, sizeof(int), cudaMemcpyDeviceToHost, st));
      LCK(cudaStreamSynchronize(st));
      if (nq) {
        const int bq = (nq + 255) / 256;
        k_cand_test<<<bq, 256, 0, st>>>(m, I(o_qpts), I(o_qptr), I(o_win), I(o_slot), lv, d_ctl, I(o_cflag),
                                        reinterpret_cast<svs_match_point*>(W + o_rec));
        svs::launch_scan(I(o_cflag), nq, I(o_cptr), st);
        k_cand_emit<<<bq, 256, 0, st>>>(Np, I(o_qptr), I(o_qpts), I(o_cflag), I(o_cptr),
                                        reinterpret_cast<const svs_match_point*>(W + o_rec), d_pts, I(o_cpt));
        LCK(cudaMemcpyAsync(&nc, I(o_cptr) + nq, sizeof(int), cudaMemcpyDeviceToHost, st));
      }
    }
    LCK(cudaGetLastError());
    LCK(cudaMemcpyAsync(&c, d_ctl, sizeof c, cudaMemcpyDeviceToHost, st));
    LCK(cudaStreamSynchronize(st));
    res->n_candidates = nc;
    if (c.no_anchor_obs) { cerr = "a candidate's anchor frame has no observation of it"; rc = SVS_ERR_INVALID; goto done; }
    if (c.bad_level) { cerr = "a candidate's anchor level is not a level of the matcher"; rc = SVS_ERR_INVALID; goto done; }
    if (c.no_slot) { cerr = "a candidate's anchor frame has no matcher slot"; rc = SVS_ERR_INVALID; goto done; }
    if (nc > mv.max_pts || nc > max_obs) { cerr = "more candidates than the matcher's max_points or the pose handle's max_obs"; rc = SVS_ERR_INVALID; goto done; }
    const double* Tlw = c.T_loop_from_w;
    k_slot_copy<<<(7 * mv.max_kf + 255) / 256, 256, 0, st>>>(mv.max_kf, mv.slot_T, mv.slot_stride, reinterpret_cast<double*>(W + o_save), 0);
    k_slot_refresh<<<(7 * V + 255) / 256, 256, 0, st>>>(V, m.pose, I(o_slot), loop, d_ctl, mv.slot_T, mv.slot_stride);
    LCK(cudaGetLastError());
    LCK(cudaStreamSynchronize(st));   // the matcher's stream reads the slots and the candidates
    refreshed = true;
    // 2 matchAndAlign
    const double I7[7] = {0, 0, 0, 1, 0, 0, 0};
    const svs_pose_params p25 = {1, 2.0, 25, -1.0, 0.00001}, p15 = {1, 2.0, 15, -1.0, 0.00001};
    const svs_match_result* d_res = nullptr;
    int nres = 0, rdev = 0;
    double T[7];
    memcpy(T, I7, sizeof T);
    for (int round = 0; round < 2; ++round) {
      rc = svs::match_device(mt, T, Tlw, d_pts, nc, round == 0 ? 10 : 4, 22, 10);
      if (rc != SVS_OK) { cerr = std::string("svs_match: ") + svs_matcher_last_error(mt); goto done; }
      svs::matcher_device_results(mt, &d_res, &nres, &rdev);
      int nm = 0;
      if (nc) {
        k_count_matched<<<1, kGate, 0, st>>>(d_res, nc, d_ctl);
        LCK(cudaGetLastError());
        LCK(cudaMemcpyAsync(&nm, &d_ctl->n_matched, sizeof(int), cudaMemcpyDeviceToHost, st));
        LCK(cudaStreamSynchronize(st));
      }
      if (round == 0) {
        res->n_matched1 = nm;
        if (nm < covis_thr) { res->stage = 1; goto done; }
      } else {
        res->n_matched2 = nm;
      }
      rc = svs_calcFastMotionOnly_matched(po, mt, cam, round == 0 ? &p25 : &p15, T, &res->lm[round]);
      if (rc != SVS_OK) { cerr = std::string("calcFastMotionOnly: ") + svs_pose_last_error(po); goto done; }
      if (round == 0) memcpy(res->T_align1, T, sizeof T);
    }
    memcpy(res->T_newloop_from_oldloop, T, sizeof T);
    if (res->n_matched2 < covis_thr) { res->stage = 2; goto done; }
    // 3 gate
    Pose7 Tn;
    memcpy(Tn.v, T, sizeof T);
    const Cam4 c4{cam->f, cam->px, cam->py, cam->b};
    k_gate<<<1, kGate, 0, st>>>(d_res, d_pts, I(o_cpt), nc, Tn, Tql, c4, mv.lv[0].w, mv.lv[0].h, m.pose, query, d_ctl, I(o_tp),
                                reinterpret_cast<double*>(W + o_tu), I(o_tl));
    LCK(cudaGetLastError());
    LCK(cudaMemcpyAsync(&c, d_ctl, sizeof c, cudaMemcpyDeviceToHost, st));
    LCK(cudaStreamSynchronize(st));
    const int nt = c.n_tracks;
    res->n_tracks = nt;
    res->num_left = c.num_left; res->num_right = c.num_right; res->num_upper = c.num_upper; res->num_lower = c.num_lower;
    if (nt > cap) { cerr = "cap is smaller than the number of tracks"; rc = SVS_ERR_INVALID; goto done; }
    if (nt) {
      LCK(cudaMemcpyAsync(track_point, I(o_tp), sizeof(int) * nt, cudaMemcpyDeviceToHost, st));
      LCK(cudaMemcpyAsync(track_uvu, W + o_tu, sizeof(double) * 3 * nt, cudaMemcpyDeviceToHost, st));
      LCK(cudaMemcpyAsync(track_level, I(o_tl), sizeof(int) * nt, cudaMemcpyDeviceToHost, st));
      LCK(cudaStreamSynchronize(st));
    }
    const int half = covis_thr / 2;
    if (nt < covis_thr) { res->stage = 3; goto done; }
    if (c.num_lower < half || c.num_upper < half || c.num_left < half || c.num_right < half) { res->stage = 4; goto done; }
    // 4 commit
    memcpy(res->T_newloop_from_w, c.T_newloop_from_w, sizeof c.T_newloop_from_w);
    rc = svs::map_add_observations(map, loop, nt, I(o_tp), reinterpret_cast<const double*>(W + o_tu), I(o_tl));
    if (rc != SVS_OK) { cerr = svs_map_last_error(map); goto done; }
    res->verified = 1;
    res->stage = 0;
  }
done:
#undef LCK
  if (rc != SVS_OK && refreshed && rc != SVS_ERR_NUMERIC) {   // a refusal leaves the slots as they were
    k_slot_copy<<<(7 * mv.max_kf + 255) / 256, 256, 0, st>>>(mv.max_kf, mv.slot_T, mv.slot_stride, reinterpret_cast<double*>(W + o_save), 1);
    cudaStreamSynchronize(st);
  }
  if (W) { cudaStreamSynchronize(st); cudaFree(W); }
  if (rc != SVS_OK) svs::map_set_error(map, cerr.c_str());
  return rc;
}
