// svs_b200.hpp -- header-only C++ host layer above the C ABI (svs_b200.h), dependency-free.
//
// Mirrors the reference's interfaces for the hot path so that a maintainer can swap the bodies
// of the corresponding ScaViSLAM methods for calls into this header (see INTEGRATION.md):
//
//   svs::OptParams / svs::Statistics   <->  ScaViSLAM::OptParams (slam_graph.hpp:36-50),
//                                           SlamGraph::Statistics (slam_graph.hpp:366-386)
//   svs::StereoGraph::optimize         <->  SlamGraph<SE3,StereoCamera,SE3XYZ_STEREO,3>::optimize
//                                           (slam_graph.cpp:319-355) = copyDataToG2o + g2o + restore
//   svs::StereoGraph::computeMarginals <->  g2o::SparseOptimizer::computeMarginals on that window
//   svs::FastGrid                      <->  ScaViSLAM::FastGrid (fast_grid.h:30-64)
//   svs::DenseTracker                  <->  ScaViSLAM::DenseTracker / GpuTracker (dense_tracking.h:40-96)
//   svs::GuidedMatcher                 <->  ScaViSLAM::GuidedMatcher<StereoCamera> (matcher.hpp:62-186)
//   svs::LinearSolverBlock6            <->  g2o::LinearSolverCSparse<Matrix6d> (slam_graph.cpp:55-60)
//
// "We do not use C++ exceptions" (reference README:295): errors come back as bool / int; the
// text is available from last_error().  There is no CPU fallback anywhere in this layer.
#ifndef SVS_B200_HPP
#define SVS_B200_HPP

#include <cmath>
#include <cstring>
#include <stdexcept>
#include <string>
#include <algorithm>
#include <utility>
#include <vector>

#include "svs_b200.h"

namespace svs {

struct SE3d {           // Sophus::SE3 as the C ABI carries it: unit quaternion (x y z w) + translation
  double q[4] = {0, 0, 0, 1};
  double t[3] = {0, 0, 0};
};

struct OptParams {      // slam_graph.hpp:36-50
  OptParams(int num_iters, bool use_robust_kernel = false, double huber_kernel_width = 1)
      : num_iters(num_iters), use_robust_kernel(use_robust_kernel), huber_kernel_width(huber_kernel_width) {}
  int num_iters;
  bool use_robust_kernel;
  double huber_kernel_width;
};

struct Statistics {     // slam_graph.hpp:366-386
  int num_frame_edges = 0, num_point_edges = 0, num_frames = 0, num_points = 0;
  double calc_time = 0;
};

// The double window handed to the optimiser: what SlamGraph::copyDataToG2o walks
// (slam_graph.cpp:985-1032).  Ids are the caller's (frame ids / point ids, any integers).
class StereoGraph {
 public:
  StereoGraph() { svs_ba_opts o{-1, 0, {0, 0, 0, 0, 0, 0}}; ok_ = svs_ba_create(&o, &h_) == SVS_OK; }
  ~StereoGraph() { if (h_) svs_ba_destroy(h_); }
  StereoGraph(const StereoGraph&) = delete;
  StereoGraph& operator=(const StereoGraph&) = delete;
  bool valid() const { return ok_; }
  svs_ba* handle() { return h_; }
  const char* last_error() const { return h_ ? svs_last_error(h_) : "svs_ba_create failed (no CUDA device)"; }

  void clear() { pose_id_.clear(); T_.clear(); fixed_.clear(); point_id_.clear(); psi_.clear(); ep_.clear(); ef_.clear();
                 ea_.clear(); obs_.clear(); info_.clear(); ci_.clear(); cj_.clear(); cT_.clear(); cL_.clear(); }
  void setCamera(double f, double px, double py, double b) { cam_ = svs_cam{f, px, py, b}; }
  // addPoseToG2o (slam_graph-impl.cpp:29-42)
  void addPose(int frame_id, const SE3d& T_me_from_w, bool fixed = false) {
    pose_id_.push_back(frame_id); push7(T_, T_me_from_w); fixed_.push_back(fixed ? 1 : 0);
  }
  // addPointToG2o (slam_graph.cpp:907-920): xyz in the anchor frame; stored as psi = invert_depth(xyz)
  void addPoint(int point_id, const double xyz_anchor[3]) {
    point_id_.push_back(point_id);
    psi_.push_back(xyz_anchor[0] / xyz_anchor[2]); psi_.push_back(xyz_anchor[1] / xyz_anchor[2]); psi_.push_back(1. / xyz_anchor[2]);
  }
  // addObsToG2o (slam_graph-impl.cpp:44-97): obs = (u, v, u_right), Lambda = diag(lambda)
  void addObs(const double obs[3], const double lambda_diag[3], int point_id, int frame_id, int anchor_id) {
    ep_.push_back(point_id); ef_.push_back(frame_id); ea_.push_back(anchor_id);
    for (int k = 0; k < 3; ++k) { obs_.push_back(obs[k]); info_.push_back(lambda_diag[k]); }
  }
  // addConstraintToG2o (slam_graph-impl.cpp:99-126): Lambda row-major 6x6
  void addConstraint(const SE3d& T_2_from_1, const double Lambda[36], int frame_id_1, int frame_id_2) {
    ci_.push_back(frame_id_1); cj_.push_back(frame_id_2); push7(cT_, T_2_from_1);
    cL_.insert(cL_.end(), Lambda, Lambda + 36);
  }

  // SlamGraph::optimize(const OptParams&, Statistics*) (slam_graph.cpp:319-355).  lambda0 = 50 and
  // 5 trials as the reference configures g2o (:338, :1073).  Note the reference never applies
  // huber_kernel_width (slam_graph-impl.cpp:86-90, delta stays 1): pass apply_huber_width = true
  // for the corrected behaviour.  Returns g2o's optimize() value.
  int optimize(const OptParams& p, Statistics* stats = nullptr, bool apply_huber_width = false) {
    if (!ok_) return -100 + SVS_ERR_NOGPU;
    std::vector<int> ep(ep_.size()), ef(ef_.size()), ea(ea_.size()), ci(ci_.size()), cj(cj_.size());
    if (!remap(ep_, point_id_, ep) || !remap(ef_, pose_id_, ef) || !remap(ea_, pose_id_, ea) ||
        !remap(ci_, pose_id_, ci) || !remap(cj_, pose_id_, cj))
      return -100 + SVS_ERR_INVALID;
    svs_ba_stats st{};
    robust_ = p.use_robust_kernel ? 1 : 0;
    delta_ = apply_huber_width ? p.huber_kernel_width : 1.0;
    opt_P_ = pose_id_.size(); opt_L_ = point_id_.size();
    const int it = svs_optimiseInnerAndOuterWindow(
        h_, (int)pose_id_.size(), T_.data(), fixed_.data(), (int)point_id_.size(), psi_.data(), (int)ep.size(), ep.data(),
        ef.data(), ea.data(), obs_.data(), info_.data(), (int)ci.size(), ci.data(), cj.data(), cT_.data(), cL_.data(), &cam_,
        p.num_iters, robust_, delta_, &st);
    if (stats && it > -100) {
      stats->num_frames = st.num_frames; stats->num_points = st.num_points;
      stats->num_point_edges = st.num_point_edges; stats->num_frame_edges = st.num_frame_edges;
      stats->calc_time = st.ms_total * 1e-3;
    }
    last_ = st;
    return it;
  }
  // restoreDataFromG2o (slam_graph.cpp:1037-1058)
  SE3d pose(size_t i) const { SE3d T; memcpy(T.q, &T_[7 * i], 32); memcpy(T.t, &T_[7 * i + 4], 24); return T; }
  void point_xyz_anchor(size_t i, double xyz[3]) const {   // invert_depth(psi)
    xyz[0] = psi_[3 * i] / psi_[3 * i + 2]; xyz[1] = psi_[3 * i + 1] / psi_[3 * i + 2]; xyz[2] = 1. / psi_[3 * i + 2];
  }
  size_t num_poses() const { return pose_id_.size(); }
  size_t num_points() const { return point_id_.size(); }
  const svs_ba_stats& last_stats() const { return last_; }

  // SparseOptimizer::computeMarginals for the window the last optimize() ran on (svs_ba_covariance): blocks of
  // (H + lambda I)^-1 at the optimised state, with the robust kernel of that call; row-major, zero for fixed poses.
  //   pose_cov  [P][36]  in addPose order;   point_cov [L][9] in psi = (x/z, y/z, 1/z), in addPoint order;
  //   pair_cov  [n][36]  Cov(x_i, x_j) for the frame ids (i, j) of pose_pairs[k].
  // Any output may be null (pair_cov only when pose_pairs is empty).  Returns false when the factor fails (the outputs
  // are zero), and when there is nothing to take them from: no optimize() on the current poses and points, an unknown
  // frame id, or an error of the C ABI (last_error(); lambda = 0 needs a fixed pose).
  bool computeMarginals(double lambda, std::vector<double>* pose_cov, std::vector<double>* point_cov,
                        const std::vector<std::pair<int, int>>& pose_pairs = {}, std::vector<double>* pair_cov = nullptr) {
    if (!ok_ || opt_P_ != pose_id_.size() || opt_L_ != point_id_.size()) return false;
    const size_t n = pose_pairs.size();
    std::vector<int> fi(n), fj(n), pi(n), pj(n);
    for (size_t k = 0; k < n; ++k) { fi[k] = pose_pairs[k].first; fj[k] = pose_pairs[k].second; }
    if (n && (!pair_cov || !remap(fi, pose_id_, pi) || !remap(fj, pose_id_, pj))) return false;
    if (pose_cov) pose_cov->assign(36 * pose_id_.size(), 0.);
    if (point_cov) point_cov->assign(9 * point_id_.size(), 0.);
    if (pair_cov) pair_cov->assign(36 * n, 0.);
    return svs_ba_covariance(h_, robust_, delta_, lambda, pose_cov ? pose_cov->data() : nullptr, (int)n, pi.data(), pj.data(),
                             n ? pair_cov->data() : nullptr, point_cov ? point_cov->data() : nullptr, nullptr) == 0;
  }

 private:
  static void push7(std::vector<double>& v, const SE3d& T) { v.insert(v.end(), T.q, T.q + 4); v.insert(v.end(), T.t, T.t + 3); }
  // id -> index through a sorted copy of the id table (ids may be sparse or hashed); a duplicate id is an error
  static bool remap(const std::vector<int>& ids, const std::vector<int>& table, std::vector<int>& out) {
    std::vector<std::pair<int, int>> sorted(table.size());
    for (size_t k = 0; k < table.size(); ++k) sorted[k] = std::make_pair(table[k], (int)k);
    std::sort(sorted.begin(), sorted.end());
    for (size_t k = 1; k < sorted.size(); ++k)
      if (sorted[k].first == sorted[k - 1].first) return false;
    for (size_t k = 0; k < ids.size(); ++k) {
      auto it = std::lower_bound(sorted.begin(), sorted.end(), std::make_pair(ids[k], 0),
                                 [](const std::pair<int, int>& a, const std::pair<int, int>& b) { return a.first < b.first; });
      if (it == sorted.end() || it->first != ids[k]) return false;
      out[k] = it->second;
    }
    return true;
  }
  svs_ba* h_ = nullptr;
  bool ok_ = false;
  svs_cam cam_{1, 0, 0, 0.5};
  std::vector<int> pose_id_, point_id_, ep_, ef_, ea_, ci_, cj_;
  std::vector<double> T_, psi_, obs_, info_, cT_, cL_;
  std::vector<unsigned char> fixed_;
  svs_ba_stats last_{};
  int robust_ = 0;
  double delta_ = 1.0;
  size_t opt_P_ = (size_t)-1, opt_L_ = (size_t)-1;   // window of the last optimize()
};

// g2o::LinearSolver<Matrix6d>::init / solve on the device (svs_chol6_*): the body of a g2o linear solver that
// keeps the rest of g2o (INTEGRATION.md shows the adapter).  solve() takes the upper triangle of A in block CCS
// (fillCCS(..., upperTriangle = true)): col_ptr[P + 1], row_idx[nnzb], blocks[nnzb * 36] column-major; x and b
// hold 6P entries.  Returns false when A is not positive definite (x is zeroed), like g2o; throws
// std::runtime_error for a malformed input or a device error, and from the constructor without a device.
class LinearSolverBlock6 {
 public:
  explicit LinearSolverBlock6(int device = -1) {
    if (svs_chol6_create(device, &h_) != SVS_OK) throw std::runtime_error("svs_chol6_create failed (no CUDA device)");
  }
  ~LinearSolverBlock6() { if (h_) svs_chol6_destroy(h_); }
  LinearSolverBlock6(const LinearSolverBlock6&) = delete;
  LinearSolverBlock6& operator=(const LinearSolverBlock6&) = delete;
  svs_chol6* handle() { return h_; }
  // LinearSolver::init(): forget the cached symbolic analysis
  void init() { check(svs_chol6_init(h_)); }
  bool solve(int P, const int* col_ptr, const int* row_idx, const double* blocks, double* x, const double* b) {
    return check(svs_chol6_solve(h_, P, col_ptr, row_idx, blocks, b, x, 0, &last_)) == 0;
  }
  // LinearSolver::solveBlocks: the P diagonal blocks of A^-1 into inv_diag [P][36] (column-major)
  bool solveBlocks(int P, const int* col_ptr, const int* row_idx, const double* blocks, double* inv_diag) {
    return check(svs_chol6_solve_blocks(h_, P, col_ptr, row_idx, blocks, inv_diag, 0, &last_inv_)) == 0;
  }
  // LinearSolver::solvePattern: blocks (r[k], c[k]) of A^-1 into out [n][36] (column-major)
  bool solvePattern(int P, const int* col_ptr, const int* row_idx, const double* blocks, int n, const int* r,
                    const int* c, double* out) {
    return check(svs_chol6_solve_pattern(h_, P, col_ptr, row_idx, blocks, n, r, c, out, 0, &last_inv_)) == 0;
  }
  const svs_chol6_stats& last_stats() const { return last_; }
  const svs_chol6_inv_stats& last_inv_stats() const { return last_inv_; }

 private:
  int check(int rc) {
    if (rc < 0) throw std::runtime_error(svs_chol6_last_error(h_));
    return rc;
  }
  svs_chol6* h_ = nullptr;
  svs_chol6_stats last_{};
  svs_chol6_inv_stats last_inv_{};
};

// ScaViSLAM::FastGrid (fast_grid.h:30-64).  Keypoints come back as flat (x, y) pairs grouped by
// cell; the quadtree content of keypoint i of cell c is i - cell_off[c].
class FastGrid {
 public:
  FastGrid(int img_w, int img_h, int num_features_per_cell, int boundary_per_cell, int fast_thr, int grid_w, int grid_h,
           int fast_min = 10, int fast_max = 40, int max_keypoints = 200000)
      : cells_((size_t)grid_w * grid_h), max_kp_(max_keypoints) {
    ok_ = svs_fast_create(-1, img_w, img_h, max_keypoints, &h_) == SVS_OK &&
          svs_fast_grid_init(img_w, img_h, num_features_per_cell, boundary_per_cell, fast_thr, grid_w, grid_h, fast_min,
                             fast_max, &grid_, cells_.data()) == SVS_OK;
  }
  ~FastGrid() { if (h_) svs_fast_destroy(h_); }
  FastGrid(const FastGrid&) = delete;
  FastGrid& operator=(const FastGrid&) = delete;
  bool valid() const { return ok_; }
  svs_fast* handle() { return h_; }
  const std::vector<svs_fast_cell>& cell_grid2d() const { return cells_; }
  // the same on an image that already lies on the device (a FramePreprocessor level)
  int detectAdaptivelyDevice(const unsigned char* d_img, int pitch, int w, int h, int trials, std::vector<int>* xy,
                             std::vector<int>* cell_off) {
    if (!ok_ || svs_fast_set_image_device(h_, d_img, pitch, w, h) != SVS_OK) return -1;
    xy->resize(2 * (size_t)max_kp_); cell_off->resize(cells_.size() + 1);
    const int n = svs_fast_detect_adaptively(h_, &grid_, cells_.data(), trials, xy->data(), max_kp_, cell_off->data());
    if (n >= 0) xy->resize(2 * (size_t)(n < max_kp_ ? n : max_kp_));
    return n;
  }
  // detectAdaptively(img, trials, qt)
  int detectAdaptively(const unsigned char* img, int pitch, int w, int h, int trials, std::vector<int>* xy,
                       std::vector<int>* cell_off) {
    if (!ok_ || svs_fast_set_image(h_, img, pitch, w, h) != SVS_OK) return -1;
    xy->resize(2 * (size_t)max_kp_); cell_off->resize(cells_.size() + 1);
    const int n = svs_fast_detect_adaptively(h_, &grid_, cells_.data(), trials, xy->data(), max_kp_, cell_off->data());
    if (n >= 0) xy->resize(2 * (size_t)(n < max_kp_ ? n : max_kp_));
    return n;
  }
  // static FastGrid::detect(img, cell_grid2d, qt)
  int detect(const unsigned char* img, int pitch, int w, int h, const std::vector<svs_fast_cell>& cells,
             std::vector<int>* xy, std::vector<int>* cell_off) {
    if (!ok_ || svs_fast_set_image(h_, img, pitch, w, h) != SVS_OK) return -1;
    xy->resize(2 * (size_t)max_kp_); cell_off->resize(cells.size() + 1);
    const int n = svs_fast_detect(h_, cells.data(), (int)cells.size(), xy->data(), max_kp_, cell_off->data());
    if (n >= 0) xy->resize(2 * (size_t)(n < max_kp_ ? n : max_kp_));
    return n;
  }

 private:
  svs_fast* h_ = nullptr;
  bool ok_ = false;
  svs_fast_grid_params grid_{};
  std::vector<svs_fast_cell> cells_;
  int max_kp_;
};

// ScaViSLAM::DenseTracker (GPU path)
class DenseTracker {
 public:
  DenseTracker(int w0, int h0, int nlevels = 3, int flags = 0) { ok_ = svs_dt_create(-1, w0, h0, nlevels, flags, &h_) == SVS_OK; }
  ~DenseTracker() { if (h_) svs_dt_destroy(h_); }
  DenseTracker(const DenseTracker&) = delete;
  DenseTracker& operator=(const DenseTracker&) = delete;
  bool valid() const { return ok_; }
  svs_dt* handle() { return h_; }
  // denseTrackingGpu(SE3 * T_cur_from_actkey)
  bool denseTrackingGpu(SE3d* T_cur_from_actkey, svs_dt_stats* stats = nullptr) {
    double T[7];
    memcpy(T, T_cur_from_actkey->q, 32); memcpy(T + 4, T_cur_from_actkey->t, 24);
    if (!ok_ || svs_dt_track(h_, T, stats) != SVS_OK) return false;
    memcpy(T_cur_from_actkey->q, T, 32); memcpy(T_cur_from_actkey->t, T + 4, 24);
    return true;
  }
  // computeDensePointCloudGpu(const SE3 & T_cur_from_actkey)
  bool computeDensePointCloudGpu(const SE3d& T_cur_from_actkey, const svs_cam* level_cams) {
    double T[7];
    memcpy(T, T_cur_from_actkey.q, 32); memcpy(T + 4, T_cur_from_actkey.t, 24);
    return ok_ && svs_dt_compute_point_cloud(h_, T, level_cams) == SVS_OK;
  }
  // frame_data_->gpu_disp_32f from a map on the device (StereoBM::disparityDevice)
  bool setDisparityDevice(const float* d_disp, int stride_floats, int w, int h) {
    return ok_ && svs_dt_set_disparity_device(h_, d_disp, stride_floats, w, h) == SVS_OK;
  }
  // GpuTracker::residualImage of one level at T_cur_from_prev (dev_residual_img[l], dense_tracking.cpp:180-188):
  // res_rgba receives w_l * h_l float4
  bool residualImage(int level, const SE3d& T_cur_from_prev, std::vector<float>* res_rgba, int w_l, int h_l) {
    double T[7];
    memcpy(T, T_cur_from_prev.q, 32); memcpy(T + 4, T_cur_from_prev.t, 24);
    res_rgba->resize((size_t)4 * w_l * h_l);
    return ok_ && svs_dt_residual_image(h_, level, T, res_rgba->data()) == SVS_OK;
  }

 private:
  svs_dt* h_ = nullptr;
  bool ok_ = false;
};

// ScaViSLAM::DenseTracker as built without SCAVISLAM_CUDA_SUPPORT (dense_tracking.cpp:222-423)
class DenseTrackerCpuVariant {
 public:
  DenseTrackerCpuVariant(int w, int h, int nlevels) { ok_ = svs_dtc_create(-1, w, h, nlevels, &h_) == SVS_OK; }
  ~DenseTrackerCpuVariant() { if (h_) svs_dtc_destroy(h_); }
  DenseTrackerCpuVariant(const DenseTrackerCpuVariant&) = delete;
  DenseTrackerCpuVariant& operator=(const DenseTrackerCpuVariant&) = delete;
  bool valid() const { return ok_; }
  svs_dtc* handle() { return h_; }
  // computeDensePointCloudCpu(T_cur_from_actkey); cam_vec = one svs_cam per pyramid level
  bool computeDensePointCloudCpu(const SE3d& T, const std::vector<svs_cam>& cam_vec) {
    const double t7[7] = {T.q[0], T.q[1], T.q[2], T.q[3], T.t[0], T.t[1], T.t[2]};
    return ok_ && svs_computeDensePointCloudCpu(h_, t7, cam_vec.data()) == SVS_OK;
  }
  // frame_data_->disp from a map on the device (StereoBM::disparityDevice)
  bool setDisparityDevice(const float* d_disp, int stride_floats) {
    return ok_ && svs_dtc_set_disparity_device(h_, d_disp, stride_floats) == SVS_OK;
  }
  // denseTrackingCpu(&T_cur_from_actkey)
  bool denseTrackingCpu(SE3d* T, const std::vector<svs_cam>& cam_vec, svs_dt_stats* stats = nullptr) {
    double t7[7] = {T->q[0], T->q[1], T->q[2], T->q[3], T->t[0], T->t[1], T->t[2]};
    if (!ok_ || svs_denseTrackingCpu(h_, cam_vec.data(), t7, stats) != SVS_OK) return false;
    for (int k = 0; k < 4; ++k) T->q[k] = t7[k];
    for (int k = 0; k < 3; ++k) T->t[k] = t7[4 + k];
    return true;
  }

 private:
  svs_dtc* h_ = nullptr;
  bool ok_ = false;
};

// ScaViSLAM::GuidedMatcher<StereoCamera>
class GuidedMatcher {
 public:
  GuidedMatcher(const std::vector<svs_match_level>& cam_vec, int max_keyframes = 8, int max_points = 8192,
                int max_keypoints = 65536)
      : nlevels_((int)cam_vec.size()), max_points_(max_points) {
    ok_ = svs_matcher_create(-1, (int)cam_vec.size(), cam_vec.data(), max_keyframes, max_points, max_keypoints, &h_) == SVS_OK;
  }
  ~GuidedMatcher() { if (h_) svs_matcher_destroy(h_); }
  GuidedMatcher(const GuidedMatcher&) = delete;
  GuidedMatcher& operator=(const GuidedMatcher&) = delete;
  bool valid() const { return ok_; }
  svs_matcher* handle() { return h_; }
  // cur_frame.disp from a map on the device (StereoBM::disparityDevice)
  bool setCurrentDisparityDevice(const float* d_disp, int pitch_floats) {
    return ok_ && svs_matcher_set_disparity_device(h_, d_disp, pitch_floats) == SVS_OK;
  }
  // feature_tree of one pyramid level = the corners FastGrid::detect* left on the device
  bool setFeatureTree(int level, FastGrid& fast_grid) { return ok_ && svs_matcher_set_features_from_fast(h_, level, fast_grid.handle()) == SVS_OK; }
  // match(keyframe_map, T_cur_from_actkey, cur_frame, feature_tree, cam_vec, actkey_id, vertex_map, ap_map,
  //       SEARCHRADIUS, thr_mean, thr_std, track_data): frames/keyframes/features are set on the handle first
  int match(const double T_cur_from_actkey[7], const double T_actkey_from_w[7], const std::vector<svs_match_point>& ap_map,
            int SEARCHRADIUS, int thr_mean, int thr_std, std::vector<svs_match_result>* track_data) {
    track_data->resize(ap_map.size());
    if (!ok_) return -1;
    return svs_match(h_, T_cur_from_actkey, T_actkey_from_w, ap_map.data(), (int)ap_map.size(), SEARCHRADIUS, thr_mean,
                     thr_std, track_data->data());
  }
  // matchAndTrack's matching (stereo_frontend.cpp:977-1050): groups = newpoint_map[actkey_id], the neighbours'
  // newpoint_map lists in strength_to_neighbors order, neighborhood_->point_list.  Returns num_obs or a negative SVS_ERR_*.
  int matchAndTrack(const double T_cur_from_actkey[7], const double T_actkey_from_w[7],
                    const std::vector<std::vector<svs_match_point>>& groups, int num_max_points,
                    std::vector<svs_match_result>* track_data, int* num_new_feat_matched, int SEARCHRADIUS = 4,
                    int thr_mean = 22, int thr_std = 10) {
    std::vector<svs_match_point> pts;
    std::vector<int> ends;
    for (const auto& g : groups) { pts.insert(pts.end(), g.begin(), g.end()); ends.push_back((int)pts.size()); }
    track_data->resize(pts.size());
    if (!ok_) return -1;
    int num_obs = 0;
    const int rc = svs_match_track(h_, T_cur_from_actkey, T_actkey_from_w, pts.data(), (int)pts.size(), (int)ends.size(),
                                   ends.data(), num_max_points, SEARCHRADIUS, thr_mean, thr_std, track_data->data(),
                                   num_new_feat_matched, &num_obs);
    return rc < 0 ? rc : num_obs;
  }
  // processMatchedPoints (stereo_frontend.cpp:834-974) on the last match, with the add flags of addNewKeyframe and the
  // result of shallWeDropNewKeyframe.  Returns the number of gated entries or a negative SVS_ERR_*.
  int processMatchedPoints(const double T_cur_from_actkey[7], const svs_cam& cam, int num_new_feat_boundary,
                           std::vector<svs_tracked_point>* tracked, svs_point_stats* stats, int add_flags[9],
                           bool* drop_keyframe, const svs_frontend_params& params = frontendDefaults()) {
    tracked->resize(max_points_);
    int drop = 0;
    const int rc = ok_ ? svs_processMatchedPoints(h_, T_cur_from_actkey, &cam, num_new_feat_boundary, &params,
                                                   tracked->data(), stats, add_flags, &drop)
                       : -1;
    tracked->resize(rc > 0 ? rc : 0);
    if (drop_keyframe) *drop_keyframe = drop == 1;
    return rc;
  }
  // addNewPoints (stereo_frontend.cpp:682-704): seeding of the first frame.  Returns the number of points or < 0.
  int addNewPoints(const svs_cam& cam, int keyframe_slot, std::vector<svs_new_point>* points,
                   std::vector<svs_match_point>* rows, const svs_frontend_params& params = frontendDefaults()) {
    return seed(1, cam, keyframe_slot, points, rows, params);
  }
  // addMorePoints (stereo_frontend.cpp:706-720) after processMatchedPoints: its tree, flags and point counts.
  int addMorePoints(const svs_cam& cam, int keyframe_slot, std::vector<svs_new_point>* points,
                    std::vector<svs_match_point>* rows, const svs_frontend_params& params = frontendDefaults()) {
    return seed(0, cam, keyframe_slot, points, rows, params);
  }
  static svs_frontend_params frontendDefaults() {
    svs_frontend_params p = SVS_FRONTEND_PARAMS_DEFAULT;
    return p;
  }

 private:
  int seed(int fresh, const svs_cam& cam, int slot, std::vector<svs_new_point>* points, std::vector<svs_match_point>* rows,
           const svs_frontend_params& params) {
    int cap = 0;
    for (int l = 0; l < nlevels_; ++l) cap += (params.num_max_points >> l) + 1;
    points->resize(cap);
    rows->resize(cap);
    const double I[7] = {0, 0, 0, 1, 0, 0, 0};
    const int rc = ok_ ? svs_addMorePoints(h_, fresh, I, &cam, slot, &params, points->data(), rows->data(), cap, nullptr) : -1;
    points->resize(rc > 0 ? rc : 0);
    rows->resize(rc > 0 ? rc : 0);
    return rc;
  }
  int nlevels_ = 0, max_points_ = 0;
  svs_matcher* h_ = nullptr;
  bool ok_ = false;
};

// StereoFrontend::PointStatistics (stereo_frontend.h:160-177)
using PointStatistics = svs_point_stats;

// StereoFrontend::shallWeDropNewKeyframe (stereo_frontend.cpp:512-528)
inline bool shallWeDropNewKeyframe(const PointStatistics& stats, const double T_cur_from_actkey[7],
                                   const svs_frontend_params& params = GuidedMatcher::frontendDefaults()) {
  return svs_shallWeDropNewKeyframe(&stats, T_cur_from_actkey, &params) == 1;
}

// ScaViSLAM::PoseOptimizerParams (pose_optimizer.h:38-58)
struct PoseOptimizerParams : svs_pose_params {
  PoseOptimizerParams(bool robust_kernel_ = true, double kernel_param_ = 1, int num_iter_ = 50, double initial_mu_ = -1) {
    robust_kernel = robust_kernel_; kernel_param = kernel_param_; num_iter = num_iter_; initial_mu = initial_mu_;
    tau = 0.00001;
  }
};

// ScaViSLAM::OptimizerStatistics (pose_optimizer.h:60-98)
struct OptimizerStatistics : svs_pose_stats {
  double rmse() const { return num_obs > 0 ? std::sqrt(chi2 / num_obs) : 0.; }
};

// ScaViSLAM::BA_SE3_XYZ_STEREO = PoseOptimizer<SE3,6,IdObs<3>,3> (pose_optimizer.h:495)
class BA_SE3_XYZ_STEREO {
 public:
  explicit BA_SE3_XYZ_STEREO(int max_obs = 16384) { ok_ = svs_pose_create(-1, max_obs, &h_) == SVS_OK; }
  ~BA_SE3_XYZ_STEREO() { if (h_) svs_pose_destroy(h_); }
  BA_SE3_XYZ_STEREO(const BA_SE3_XYZ_STEREO&) = delete;
  BA_SE3_XYZ_STEREO& operator=(const BA_SE3_XYZ_STEREO&) = delete;
  bool valid() const { return ok_; }
  svs_pose* handle() { return h_; }
  // calcFastMotionOnly(obs_list, prediction(cam), ba_params, &frame, &point_list); throws where the reference does
  OptimizerStatistics calcFastMotionOnly(const std::vector<int>& obs_point_id, const std::vector<double>& obs_uvu,
                                         const svs_cam& cam, const PoseOptimizerParams& ba_params, SE3d* frame,
                                         const std::vector<double>& point_list_xyz) {
    OptimizerStatistics st{};
    double T[7] = {frame->q[0], frame->q[1], frame->q[2], frame->q[3], frame->t[0], frame->t[1], frame->t[2]};
    const int rc = ok_ ? svs_calcFastMotionOnly(h_, (int)obs_point_id.size(), obs_point_id.data(), obs_uvu.data(),
                                                (int)(point_list_xyz.size() / 3), point_list_xyz.data(), &cam, &ba_params,
                                                T, &st)
                       : SVS_ERR_NOGPU;
    if (rc != SVS_OK) throw std::runtime_error(ok_ ? svs_pose_last_error(h_) : "no CUDA device");
    for (int k = 0; k < 4; ++k) frame->q[k] = T[k];
    for (int k = 0; k < 3; ++k) frame->t[k] = T[4 + k];
    return st;
  }
  // the same on the TrackData the matcher left on the device
  OptimizerStatistics calcFastMotionOnly(GuidedMatcher& matcher, const svs_cam& cam, const PoseOptimizerParams& ba_params,
                                         SE3d* frame) {
    OptimizerStatistics st{};
    double T[7] = {frame->q[0], frame->q[1], frame->q[2], frame->q[3], frame->t[0], frame->t[1], frame->t[2]};
    const int rc = ok_ ? svs_calcFastMotionOnly_matched(h_, matcher.handle(), &cam, &ba_params, T, &st) : SVS_ERR_NOGPU;
    if (rc != SVS_OK) throw std::runtime_error(ok_ ? svs_pose_last_error(h_) : "no CUDA device");
    for (int k = 0; k < 4; ++k) frame->q[k] = T[k];
    for (int k = 0; k < 3; ++k) frame->t[k] = T[4 + k];
    return st;
  }

 private:
  svs_pose* h_ = nullptr;
  bool ok_ = false;
};

// FrameGrabber::preprocessing (frame_grabber.cpp:287-336): pyramids and derivative images, kept on the device
class FramePreprocessor {
 public:
  FramePreprocessor(int w, int h, int nlevels) { ok_ = svs_prep_create(-1, w, h, nlevels, &h_) == SVS_OK; }
  ~FramePreprocessor() { if (h_) svs_prep_destroy(h_); }
  FramePreprocessor(const FramePreprocessor&) = delete;
  FramePreprocessor& operator=(const FramePreprocessor&) = delete;
  bool valid() const { return ok_; }
  svs_prep* handle() { return h_; }
  bool preprocessing(const unsigned char* left, int pitch) { return ok_ && svs_prep_process(h_, left, pitch) == SVS_OK; }
  // device pointers of one level: hand them to svs_fast_set_image_device / svs_dt_set_images_device / ...
  struct Level { int w, h, pitch_u8, stride_f32; const unsigned char* u8; const float *f32, *dx, *dy; };
  bool level(int l, Level* out) {
    return ok_ && svs_prep_level(h_, l, &out->w, &out->h, &out->u8, &out->pitch_u8, &out->f32, &out->dx, &out->dy,
                                 &out->stride_f32) == SVS_OK;
  }

 private:
  svs_prep* h_ = nullptr;
  bool ok_ = false;
};

// StereoFrontend::calcDisparityCpu (stereo_frontend.cpp:620-653): cv::StereoBM with the reference's settings, the
// map kept on the device (svs_stereo_* in svs_b200.h states the semantics)
class StereoBM {
 public:
  StereoBM(int w, int h, int num_disparities = 32) { ok_ = svs_stereo_create(-1, w, h, num_disparities, &h_) == SVS_OK; }
  ~StereoBM() { if (h_) svs_stereo_destroy(h_); }
  StereoBM(const StereoBM&) = delete;
  StereoBM& operator=(const StereoBM&) = delete;
  bool valid() const { return ok_; }
  svs_stereo* handle() { return h_; }
  // left / right uint8 images; *_on_device: the image is device memory (e.g. FramePreprocessor level 0)
  bool calcDisparity(const unsigned char* left, int left_pitch, const unsigned char* right, int right_pitch,
                     bool left_on_device = false, bool right_on_device = false) {
    return ok_ && svs_stereo_compute(h_, left, left_pitch, left_on_device, right, right_pitch, right_on_device) == SVS_OK;
  }
  // the map on the device, for DenseTracker / DenseTrackerCpuVariant / GuidedMatcher ::set*DisparityDevice
  bool disparityDevice(const float** d_disp, int* stride_floats) {
    return ok_ && svs_stereo_disparity(h_, d_disp, stride_floats) == SVS_OK;
  }
  bool disparity(float* out) { return ok_ && svs_stereo_get(h_, out) == SVS_OK; }   // w*h, tightly packed
  const char* last_error() const { return svs_stereo_last_error(h_); }

 private:
  svs_stereo* h_ = nullptr;
  bool ok_ = false;
};

// SlamGraph::computeConstraint (slam_graph.cpp:785-846) for a batch of pose pairs
class ConstraintBuilder {
 public:
  ConstraintBuilder() { ok_ = svs_constraints_create(-1, &h_) == SVS_OK; }
  ~ConstraintBuilder() { if (h_) svs_constraints_destroy(h_); }
  ConstraintBuilder(const ConstraintBuilder&) = delete;
  ConstraintBuilder& operator=(const ConstraintBuilder&) = delete;
  bool valid() const { return ok_; }
  const char* last_error() const { return svs_constraints_last_error(h_); }
  // poses [P][7]; feature tables as CSR (ascending point ids); per point its anchor pose index and xyz_anchor
  bool computeConstraints(const std::vector<double>& T_me_from_world, const std::vector<int>& feat_ptr,
                          const std::vector<int>& feat_point, const std::vector<int>& point_anchor,
                          const std::vector<double>& xyz_anchor, const std::vector<int>& v1, const std::vector<int>& v2,
                          std::vector<double>* T_1_from_2, std::vector<double>* Lambda, std::vector<int>* visibility_strength) {
    const int n = (int)v1.size();
    T_1_from_2->resize(7 * (size_t)n); Lambda->resize(36 * (size_t)n); visibility_strength->resize(n);
    return ok_ && v2.size() == v1.size() &&
           svs_computeConstraint_batch(h_, (int)(T_me_from_world.size() / 7), T_me_from_world.data(), feat_ptr.data(),
                                       feat_point.data(), (int)point_anchor.size(), point_anchor.data(), xyz_anchor.data(), n,
                                       v1.data(), v2.data(), T_1_from_2->data(), Lambda->data(),
                                       visibility_strength->data()) == SVS_OK;
  }

 private:
  svs_constraints* h_ = nullptr;
  bool ok_ = false;
};

// PlaceRecognizer::addLocation (placerecognizer.cpp:206-324) after the caller's SURF step; semantics: svs_place
struct DetectedLoop {   // placerecognizer.h
  int query_keyframe_id = -1, loop_keyframe_id = -1;
  SE3d T_query_from_loop;
};

class PlaceRecognizer {
 public:
  // words [W][64] (the vocabulary the reference reads from surfwords10000.png), cam = the stereo camera
  PlaceRecognizer(const std::vector<float>& words, const svs_cam& cam, int device = -1) {
    ok_ = words.size() >= 64 && svs_place_create(device, (int)(words.size() / 64), words.data(), &cam, &h_) == SVS_OK;
  }
  ~PlaceRecognizer() { if (h_) svs_place_destroy(h_); }
  PlaceRecognizer(const PlaceRecognizer&) = delete;
  PlaceRecognizer& operator=(const PlaceRecognizer&) = delete;
  bool valid() const { return ok_; }
  const char* last_error() const { return h_ ? svs_place_last_error(h_) : "no handle"; }
  svs_place_params params = SVS_PLACE_PARAMS_DEFAULT;
  const svs_place_result& last_result() const { return res_; }

  // descriptors [n][64], uvu [n][3] = (u, v, u - disparity) of the rows with a disparity.  Returns false on a refused
  // input or a device error; *loop is written when the check finds a loop (more than 30 inliers), as
  // geometricCheck's monitor.addLoop would receive it.
  bool addLocation(int keyframe_id, const std::vector<float>& descriptors, const std::vector<double>& uvu,
                   const std::vector<int>& exclude_set, bool do_loop_detection, DetectedLoop* loop,
                   std::vector<int>* inlier_query = nullptr, std::vector<int>* inlier_train = nullptr) {
    const int n = (int)(descriptors.size() / 64);
    if (!ok_ || descriptors.size() != 64 * (size_t)n || uvu.size() != 3 * (size_t)n) return false;
    std::vector<int> iq((size_t)std::max(n, 1)), it((size_t)std::max(n, 1));
    if (svs_place_add_location(h_, keyframe_id, n, descriptors.data(), uvu.data(), do_loop_detection ? 1 : 0,
                               (int)exclude_set.size(), exclude_set.data(), &params, &res_, iq.data(), it.data()) != SVS_OK)
      return false;
    if (inlier_query) inlier_query->assign(iq.begin(), iq.begin() + res_.num_inliers);
    if (inlier_train) inlier_train->assign(it.begin(), it.begin() + res_.num_inliers);
    if (loop && res_.loop_found) {
      loop->query_keyframe_id = keyframe_id;
      loop->loop_keyframe_id = res_.best_keyframe_id;
      std::memcpy(loop->T_query_from_loop.q, res_.T_query_from_loop, sizeof(double) * 4);
      std::memcpy(loop->T_query_from_loop.t, res_.T_query_from_loop + 4, sizeof(double) * 3);
    }
    return true;
  }

 private:
  svs_place* h_ = nullptr;
  bool ok_ = false;
  svs_place_result res_{};
};

// The part of SlamGraph the optimiser reads, kept on the device; copyDataToG2o as kernels (slam_graph.cpp:907-1032)
class DeviceMap {
 public:
  DeviceMap() { ok_ = svs_map_create(-1, &h_) == SVS_OK; }
  ~DeviceMap() { if (h_) svs_map_destroy(h_); }
  DeviceMap(const DeviceMap&) = delete;
  DeviceMap& operator=(const DeviceMap&) = delete;
  bool valid() const { return ok_; }
  svs_map* handle() { return h_; }
  const char* last_error() const { return svs_map_last_error(h_); }
  // vertex_table_ / point_table_ / feature tables as flat arrays (slam_graph.hpp:65-137): poses [V][7], per point its
  // anchor vertex and xyz_anchor, vis_set + feature_table as CSR over the points (centre (u,v,u_r) and pyramid level)
  bool set(const std::vector<double>& T_me_from_world, const std::vector<int>& point_anchor, const std::vector<double>& xyz_anchor,
           const std::vector<int>& vis_ptr, const std::vector<int>& vis_pose, const std::vector<double>& feat_center,
           const std::vector<int>& feat_level) {
    V_ = (int)(T_me_from_world.size() / 7); Np_ = (int)point_anchor.size();
    return ok_ && svs_map_set(h_, V_, T_me_from_world.data(), Np_, point_anchor.data(), xyz_anchor.data(), vis_ptr.data(),
                              vis_pose.data(), feat_center.data(), feat_level.data()) == SVS_OK;
  }
  // copyDataToG2o (slam_graph.cpp:985-1032) into `graph`'s bundle adjuster; returns the number of edges, < 0 on error
  int copyDataToG2o(svs_ba* ba, const std::vector<int>& window_vertex, const std::vector<int>& active_point, const svs_cam& cam,
                    const std::vector<int>& c_i = {}, const std::vector<int>& c_j = {}, const std::vector<double>& c_T = {},
                    const std::vector<double>& c_Lambda = {}) {
    int E = 0;
    const int rc = ok_ ? svs_ba_set_problem_from_map(ba, h_, (int)window_vertex.size(), window_vertex.data(), nullptr,
                                                     (int)active_point.size(), active_point.data(), (int)c_i.size(), c_i.data(),
                                                     c_j.data(), c_T.data(), c_Lambda.data(), &cam, &E)
                       : SVS_ERR_NOGPU;
    return rc == SVS_OK ? E : rc;
  }
  // restoreDataFromG2o (slam_graph.cpp:1037-1058), device to device
  bool restoreDataFromG2o(svs_ba* ba) { return ok_ && svs_map_absorb(h_, ba) == SVS_OK; }
  bool updatePoses(const std::vector<int>& vertex, const std::vector<double>& T) {
    return ok_ && svs_map_update_poses(h_, (int)vertex.size(), vertex.data(), T.data()) == SVS_OK;
  }
  bool updatePoints(const std::vector<int>& point, const std::vector<double>& xyz_anchor) {
    return ok_ && svs_map_update_points(h_, (int)point.size(), point.data(), xyz_anchor.data()) == SVS_OK;
  }
  // the pose graph: per vertex its neighbours, strongest first (Vertex::neighbor_ids_ordered_by_strength), and per
  // directed entry the marginalised constraint of the edge table (both payload vectors may be empty)
  bool setGraph(const std::vector<int>& nbr_ptr, const std::vector<int>& nbr_id, const std::vector<double>& nbr_T = {},
                const std::vector<double>& nbr_Lambda = {}) {
    nn_ = (int)nbr_id.size();
    return ok_ && svs_map_set_graph(h_, nbr_ptr.data(), nbr_id.data(), nbr_T.empty() ? nullptr : nbr_T.data(),
                                    nbr_Lambda.empty() ? nullptr : nbr_Lambda.data()) == SVS_OK;
  }
  // computeInitialDoubleWin + computeActivePointsAndExtendOuterWindow + the pair loop of copyContraintsToG2o
  // (slam_graph.cpp:556-663, 938-981): what prepareForOptimization (:290-311) hands to copyDataToG2o
  struct DoubleWindow {
    std::vector<int> window_vertex, active_point, c_i, c_j;
    std::vector<unsigned char> inner;
    std::vector<double> c_T, c_Lambda;
  };
  bool computeDoubleWindow(int root_id, int inner_window_size, int double_window_size, DoubleWindow* w) {
    if (!ok_) return false;
    const int capC = nn_ > 0 ? nn_ : 1;
    w->window_vertex.resize(V_); w->inner.resize(V_); w->active_point.resize(Np_ > 0 ? Np_ : 1);
    w->c_i.resize(capC); w->c_j.resize(capC); w->c_T.resize(7 * (size_t)capC); w->c_Lambda.resize(36 * (size_t)capC);
    int P = 0, L = 0, C = 0;
    if (svs_map_select_window(h_, root_id, inner_window_size, double_window_size, V_, &P, w->window_vertex.data(), w->inner.data(),
                              (int)w->active_point.size(), &L, w->active_point.data(), capC, &C, w->c_i.data(), w->c_j.data(),
                              w->c_T.data(), w->c_Lambda.data()) != SVS_OK)
      return false;
    w->window_vertex.resize(P); w->inner.resize(P); w->active_point.resize(L);
    w->c_i.resize(C); w->c_j.resize(C); w->c_T.resize(7 * (size_t)C); w->c_Lambda.resize(36 * (size_t)C);
    return true;
  }
  // addKeyframe (slam_graph.cpp:144-186): returns the index of the new vertex, < 0 on error
  int addKeyframe(int oldkey_id, const double T_newkey_from_oldkey[7], const std::vector<int>& new_anchor,
                  const std::vector<double>& new_xyz_anchor, const std::vector<double>& new_anchor_center,
                  const std::vector<int>& new_anchor_level, const std::vector<double>& new_center, const std::vector<int>& new_level,
                  const std::vector<int>& track_point, const std::vector<double>& track_center, const std::vector<int>& track_level) {
    if (!ok_) return SVS_ERR_NOGPU;
    int v = -1, q = -1;
    const int rc = svs_map_add_keyframe(h_, oldkey_id, T_newkey_from_oldkey, (int)new_anchor.size(), new_anchor.data(),
                                        new_xyz_anchor.data(), new_anchor_center.data(), new_anchor_level.data(), new_center.data(),
                                        new_level.data(), (int)track_point.size(), track_point.data(), track_center.data(),
                                        track_level.data(), &v, &q);
    if (rc != SVS_OK) return rc;
    V_ += 1; Np_ += (int)new_anchor.size(); nn_ = 0;
    return v;
  }
  // the pose graph with strengths and constraints (svs_map_set_pose_graph): what the growth calls below extend
  struct PoseGraph { std::vector<int> nbr_ptr, nbr_id, nbr_strength; std::vector<double> nbr_T, nbr_Lambda; };
  bool setPoseGraph(const PoseGraph& g) {
    if (!ok_ || svs_map_set_pose_graph(h_, g.nbr_ptr.data(), g.nbr_id.data(), g.nbr_strength.data(), g.nbr_T.data(),
                                       g.nbr_Lambda.data()) != SVS_OK)
      return false;
    nn_ = (int)g.nbr_id.size();
    return true;
  }
  // the pose graph as it lies on the device (svs_map_get_graph)
  bool poseGraph(PoseGraph* g) {
    int nn = 0;
    if (!ok_ || svs_map_get_graph(h_, 0, &nn, nullptr, nullptr, nullptr, nullptr, nullptr) != SVS_OK) return false;
    const size_t cap = nn > 0 ? (size_t)nn : 1;
    g->nbr_ptr.resize((size_t)V_ + 1); g->nbr_id.resize(cap); g->nbr_strength.resize(cap);
    g->nbr_T.resize(7 * cap); g->nbr_Lambda.resize(36 * cap);
    if (svs_map_get_graph(h_, nn, &nn, g->nbr_ptr.data(), g->nbr_id.data(), g->nbr_strength.data(), g->nbr_T.data(),
                          g->nbr_Lambda.data()) != SVS_OK)
      return false;
    g->nbr_id.resize(nn); g->nbr_strength.resize(nn); g->nbr_T.resize(7 * (size_t)nn); g->nbr_Lambda.resize(36 * (size_t)nn);
    return true;
  }
  // the whole of addKeyframe (slam_graph.cpp:144-186) with computeStrength and addNewEdges(LOCAL) on the device graph
  // (svs_map_add_keyframe_graph); `table` (may be NULL) receives the (vertex, strength) rows.  Returns the index of the
  // new vertex, < 0 on error.
  int addKeyframe(int oldkey_id, const double T_newkey_from_oldkey[7], const std::vector<int>& new_anchor,
                  const std::vector<double>& new_xyz_anchor, const std::vector<double>& new_anchor_center,
                  const std::vector<int>& new_anchor_level, const std::vector<double>& new_center, const std::vector<int>& new_level,
                  const std::vector<int>& track_point, const std::vector<double>& track_center, const std::vector<int>& track_level,
                  int covis_thr, int width, int height, std::vector<int>* table = nullptr, int* n_edges = nullptr) {
    if (!ok_) return SVS_ERR_NOGPU;
    int v = -1, q = -1, nt = 0, ne = 0;
    std::vector<int> rows(2 * (size_t)(V_ > 0 ? V_ : 1));
    const int rc = svs_map_add_keyframe_graph(h_, oldkey_id, T_newkey_from_oldkey, (int)new_anchor.size(), new_anchor.data(),
                                              new_xyz_anchor.data(), new_anchor_center.data(), new_anchor_level.data(),
                                              new_center.data(), new_level.data(), (int)track_point.size(), track_point.data(),
                                              track_center.data(), track_level.data(), covis_thr, width, height, &v, &q, &nt,
                                              rows.data(), &ne);
    if (rc != SVS_OK) return rc;
    V_ += 1; Np_ += (int)new_anchor.size(); nn_ += 2 * ne;
    if (table) table->assign(rows.begin(), rows.begin() + 2 * (size_t)nt);
    if (n_edges) *n_edges = ne;
    return v;
  }
  // registerKeyframes' METRIC edges and addLoopClosure's APPEARANCE edge (svs_map_add_edges): (v1[k], v2[k]) with
  // strength[k], computeConstraint(v1, v2) with moved_vertex (or -1) placed at T_moved_from_w
  bool addEdges(const std::vector<int>& v1, const std::vector<int>& v2, const std::vector<int>& strength, int moved_vertex = -1,
                const double* T_moved_from_w = nullptr) {
    if (!ok_ || v1.size() != v2.size() || v1.size() != strength.size()) return false;
    if (svs_map_add_edges(h_, (int)v1.size(), v1.data(), v2.data(), strength.data(), moved_vertex, T_moved_from_w) != SVS_OK)
      return false;
    nn_ += 2 * (int)v1.size();
    return true;
  }
  // prepareForOptimization(root_id, loop_id) (slam_graph.cpp:290-310; svs_map_prepare_for_optimization): the window of
  // computeDoubleWindow, reinitializePoses, unmargPosesEnteringInnerW and margPosesLeftInnerWindow on the device.  *w
  // receives the window with its constraints read after the marginalisation.  Returns whether the window holds >= 2
  // frames (the reference's return value); throws std::runtime_error on a refused call.
  bool prepareForOptimization(int root_id, int loop_id, int inner_window_size, int double_window_size, DoubleWindow* w) {
    if (!ok_) throw std::runtime_error("no CUDA device");
    const int capC = nn_ > 0 ? nn_ : 1;
    w->window_vertex.resize(V_); w->inner.resize(V_); w->active_point.resize(Np_ > 0 ? Np_ : 1);
    w->c_i.resize(capC); w->c_j.resize(capC); w->c_T.resize(7 * (size_t)capC); w->c_Lambda.resize(36 * (size_t)capC);
    int P = 0, L = 0, C = 0, do_opt = 0;
    const int rc = svs_map_prepare_for_optimization(h_, root_id, loop_id, inner_window_size, double_window_size, &do_opt, V_, &P,
                                                    w->window_vertex.data(), w->inner.data(), (int)w->active_point.size(), &L,
                                                    w->active_point.data(), capC, &C, w->c_i.data(), w->c_j.data(), w->c_T.data(),
                                                    w->c_Lambda.data());
    if (rc != SVS_OK) throw std::runtime_error(std::string("svs_map_prepare_for_optimization: ") + last_error());
    w->window_vertex.resize(P); w->inner.resize(P); w->active_point.resize(L);
    w->c_i.resize(C); w->c_j.resize(C); w->c_T.resize(7 * (size_t)C); w->c_Lambda.resize(36 * (size_t)C);
    return do_opt != 0;
  }
  // the window of the last prepare (window_type[V]: 0 outside, 1 INNER, 2 OUTER) and Edge::is_marginalized of every
  // directed entry in poseGraph's order (svs_map_get_window_state); throws std::runtime_error on a refused call
  void windowState(std::vector<unsigned char>* window_type, std::vector<unsigned char>* marginalized) {
    if (!ok_) throw std::runtime_error("no CUDA device");
    int nn = 0;
    if (svs_map_get_window_state(h_, 0, &nn, nullptr, nullptr) != SVS_OK)
      throw std::runtime_error(std::string("svs_map_get_window_state: ") + last_error());
    window_type->resize(V_ > 0 ? V_ : 1); marginalized->resize(nn > 0 ? nn : 1);
    if (svs_map_get_window_state(h_, nn, &nn, window_type->data(), marginalized->data()) != SVS_OK)
      throw std::runtime_error(std::string("svs_map_get_window_state: ") + last_error());
    window_type->resize(V_); marginalized->resize(nn);
  }
  // Backend::globalLoopClosure (backend.cpp:830-1001) on this map; semantics: svs_globalLoopClosure.  The matcher holds
  // the loop keyframe as its current frame and the keyframe pyramids in the slots vertex_slot names.  Returns true when
  // the loop was verified and the map grew; *res (when given) holds the counts of every stage reached, *tracks the gated
  // tracks.  Throws std::runtime_error on a refused call and where the reference throws (a NaN residual).
  struct LoopTracks { std::vector<int> point, level; std::vector<double> uvu; };
  bool globalLoopClosure(GuidedMatcher& matcher, BA_SE3_XYZ_STEREO& ba, const svs_cam& cam, int covis_thr, int query_id,
                         int loop_id, const SE3d& T_query_from_loop, const std::vector<int>& window_vertex,
                         const std::vector<int>& vertex_slot, svs_loop_result* res = nullptr, LoopTracks* tracks = nullptr) {
    if (!ok_) throw std::runtime_error("no CUDA device");
    if ((int)vertex_slot.size() != V_) throw std::runtime_error("vertex_slot must name a slot (or -1) for every vertex");
    const double T[7] = {T_query_from_loop.q[0], T_query_from_loop.q[1], T_query_from_loop.q[2], T_query_from_loop.q[3],
                         T_query_from_loop.t[0], T_query_from_loop.t[1], T_query_from_loop.t[2]};
    const int cap = Np_ > 0 ? Np_ : 1;   // tracks <= candidates <= points
    std::vector<int> tp(cap), tl(cap);
    std::vector<double> tu(3 * (size_t)cap);
    svs_loop_result r{};
    const int rc = svs_globalLoopClosure(h_, matcher.handle(), ba.handle(), &cam, covis_thr, query_id, loop_id, T,
                                         (int)window_vertex.size(), window_vertex.data(), vertex_slot.data(), &r, cap, tp.data(),
                                         tu.data(), tl.data());
    if (res) *res = r;
    if (rc != SVS_OK) throw std::runtime_error(svs_map_last_error(h_));
    if (tracks) {
      const int n = (r.stage == 0 || r.stage >= 3) ? r.n_tracks : 0;
      tracks->point.assign(tp.begin(), tp.begin() + n);
      tracks->level.assign(tl.begin(), tl.begin() + n);
      tracks->uvu.assign(tu.begin(), tu.begin() + 3 * (size_t)n);
    }
    return r.verified != 0;
  }

  // Backend::localRegisterFrame (backend.cpp:549-784) on this map; semantics: svs_localRegisterFrame.  The pose graph
  // must be set (setGraph); the matcher holds the root keyframe as its current frame and the keyframe pyramids in the
  // slots vertex_slot names.  Returns true when the frame was registered and the map grew; *res (when given) holds the
  // counts of every stage reached, *stats the stats table, *tracks the gated tracks.  Throws std::runtime_error on a
  // refused call (the missing pose graph included) and where the reference throws (a NaN residual).
  struct RegisterTracks { std::vector<int> point, level, committed; std::vector<double> uvu; };
  bool localRegisterFrame(GuidedMatcher& matcher, BA_SE3_XYZ_STEREO& ba, const svs_cam& cam, int covis_thr, int root_id,
                          const std::vector<int>& window_vertex, const std::vector<int>& vertex_slot,
                          svs_register_result* res = nullptr, std::vector<svs_register_stats>* stats = nullptr,
                          RegisterTracks* tracks = nullptr) {
    if (!ok_) throw std::runtime_error("no CUDA device");
    if ((int)vertex_slot.size() != V_) throw std::runtime_error("vertex_slot must name a slot (or -1) for every vertex");
    const int cs = V_ > 0 ? V_ : 1, ct = Np_ > 0 ? Np_ : 1;   // stats <= vertices, tracks <= candidates <= points
    std::vector<svs_register_stats> st(cs);
    std::vector<int> tp(ct), tl(ct), tc(ct);
    std::vector<double> tu(3 * (size_t)ct);
    svs_register_result r{};
    const int rc = svs_localRegisterFrame(h_, matcher.handle(), ba.handle(), &cam, covis_thr, root_id, (int)window_vertex.size(),
                                          window_vertex.data(), vertex_slot.data(), &r, cs, st.data(), ct, tp.data(), tu.data(),
                                          tl.data(), tc.data());
    if (res) *res = r;
    if (rc != SVS_OK) throw std::runtime_error(svs_map_last_error(h_));
    const bool gated = r.stage == 0 || r.stage == 4;
    if (stats) stats->assign(st.begin(), st.begin() + (gated ? r.n_stats : 0));
    if (tracks) {
      const int n = gated ? r.n_tracks : 0;
      tracks->point.assign(tp.begin(), tp.begin() + n);
      tracks->level.assign(tl.begin(), tl.begin() + n);
      tracks->committed.assign(tc.begin(), tc.begin() + n);
      tracks->uvu.assign(tu.begin(), tu.begin() + 3 * (size_t)n);
    }
    return r.registered != 0;
  }
  bool get(std::vector<double>* T_me_from_world, std::vector<double>* xyz_anchor) {
    T_me_from_world->resize(7 * (size_t)V_); xyz_anchor->resize(3 * (size_t)(Np_ > 0 ? Np_ : 1));
    const bool r = ok_ && svs_map_get(h_, T_me_from_world->data(), xyz_anchor->data()) == SVS_OK;
    xyz_anchor->resize(3 * (size_t)Np_);
    return r;
  }

 private:
  svs_map* h_ = nullptr;
  bool ok_ = false;
  int V_ = 0, Np_ = 0, nn_ = 0;
};

}  // namespace svs
#endif
