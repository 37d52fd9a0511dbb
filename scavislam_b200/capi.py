"""ctypes binding of libsvsb200.so (the C ABI declared in include/svs_b200.h).

This is how the tests and bench.py reach the product: through the same C ABI a
maintainer of the reference would bind from C++ (INTEGRATION.md).  There is no
CPU fallback here: if the library is missing or no CUDA device is present the
calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsvsb200.so")
_LIB = None

c_dp = C.POINTER(C.c_double)
c_ip = C.POINTER(C.c_int)
c_up = C.POINTER(C.c_ubyte)

SVS_BA_MAX_ITERS = 64
SVS_BA_SKIP_SELF_ANCHOR_HESSIAN = 1
SVS_BA_NATURAL_ORDER = 2


class SvsCam(C.Structure):
    _fields_ = [("f", C.c_double), ("px", C.c_double), ("py", C.c_double), ("b", C.c_double)]


class SvsBaOpts(C.Structure):
    _fields_ = [("device", C.c_int), ("flags", C.c_int), ("reserved", C.c_int * 6)]


class SvsBaStats(C.Structure):
    _fields_ = [("iterations", C.c_int), ("trials_total", C.c_int),
                ("chi2_init", C.c_double), ("chi2_final", C.c_double), ("lambda_final", C.c_double),
                ("chi2_iter", C.c_double * SVS_BA_MAX_ITERS), ("lambda_iter", C.c_double * SVS_BA_MAX_ITERS),
                ("trials_iter", C.c_int * SVS_BA_MAX_ITERS),
                ("num_frames", C.c_int), ("num_points", C.c_int),
                ("num_point_edges", C.c_int), ("num_frame_edges", C.c_int),
                ("nnzb_S", C.c_int), ("nnzb_L", C.c_int), ("max_track", C.c_int),
                ("ms_total", C.c_float), ("ms_build", C.c_float), ("ms_solve", C.c_float),
                ("ms_update", C.c_float), ("ms_control", C.c_float), ("launches", C.c_int)]

    def as_dict(self):
        n = max(self.iterations, 0)
        d = {k: getattr(self, k) for k, _ in self._fields_ if k not in ("chi2_iter", "lambda_iter", "trials_iter")}
        d["chi2_iter"] = list(self.chi2_iter[:n])
        d["lambda_iter"] = list(self.lambda_iter[:n])
        d["trials_iter"] = list(self.trials_iter[:n])
        return d


class SvsChol6Stats(C.Structure):
    _fields_ = [("P", C.c_int), ("nnzb_A", C.c_int), ("nnzb_L", C.c_int), ("nbranch", C.c_int), ("general", C.c_int),
                ("symbolic_reused", C.c_int), ("ms", C.c_float)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class SvsChol6InvStats(C.Structure):
    _fields_ = [("P", C.c_int), ("nnzb_A", C.c_int), ("nnzb_L", C.c_int), ("nbranch", C.c_int), ("general", C.c_int),
                ("symbolic_reused", C.c_int), ("n_in_pattern", C.c_int), ("n_cols_solved", C.c_int), ("ms", C.c_float)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class SvsBaCovStats(C.Structure):
    _fields_ = [("P", C.c_int), ("L", C.c_int), ("nnzb_L", C.c_int), ("nbranch", C.c_int), ("general", C.c_int),
                ("n_pairs_in_pattern", C.c_int), ("n_cols_solved", C.c_int), ("ms", C.c_float)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class SvsBaGradStats(C.Structure):
    _fields_ = [("P", C.c_int), ("L", C.c_int), ("E", C.c_int), ("nnzb_L", C.c_int), ("nbranch", C.c_int),
                ("general", C.c_int), ("ms", C.c_float)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class SvsBaGradOut(C.Structure):
    _fields_ = [("dL_dobs", C.c_void_p), ("dL_dinfo", C.c_void_p), ("dL_dcT", C.c_void_p), ("dL_dcLambda", C.c_void_p),
                ("dL_dcam", C.c_void_p)]


class SvsFastCell(C.Structure):
    _fields_ = [("u0", C.c_int), ("u1", C.c_int), ("v0", C.c_int), ("v1", C.c_int), ("thr", C.c_int)]


class SvsFastGridParams(C.Structure):
    _fields_ = [("grid_w", C.c_int), ("grid_h", C.c_int), ("fast_min", C.c_int), ("fast_max", C.c_int),
                ("min_inner", C.c_int), ("min_outer", C.c_int), ("max_inner", C.c_int), ("max_outer", C.c_int)]


SVS_DT_MAX_LEVELS = 8
SVS_DT_EXACT_BILINEAR = 1


class SvsDtStats(C.Structure):
    _fields_ = [("chi2", C.c_double * SVS_DT_MAX_LEVELS), ("passes", C.c_int * SVS_DT_MAX_LEVELS),
                ("launches", C.c_int), ("ms_total", C.c_float)]


class SvsPoseParams(C.Structure):
    _fields_ = [("robust_kernel", C.c_int), ("kernel_param", C.c_double), ("num_iter", C.c_int),
                ("initial_mu", C.c_double), ("tau", C.c_double)]


class SvsPoseStats(C.Structure):
    _fields_ = [("initial_chi2", C.c_double), ("chi2", C.c_double), ("max_err", C.c_double), ("num_obs", C.c_int),
                ("iterations", C.c_int), ("trials", C.c_int), ("ms", C.c_float)]


class SvsPoseGradStats(C.Structure):
    _fields_ = [("num_obs", C.c_int), ("npoints", C.c_int), ("ms", C.c_float)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class SvsMatchLevel(C.Structure):
    _fields_ = [("w", C.c_int), ("h", C.c_int), ("f", C.c_double), ("px", C.c_double), ("py", C.c_double)]


class SvsMatchPoint(C.Structure):
    _fields_ = [("keyframe", C.c_int), ("anchor_level", C.c_int), ("xyz_anchor", C.c_double * 3),
                ("anchor_obs_pyr", C.c_double * 2)]


class SvsMatchResult(C.Structure):
    _fields_ = [("predicted", C.c_int), ("textured", C.c_int), ("matched", C.c_int), ("n_candidates", C.c_int),
                ("index", C.c_int), ("min_dist", C.c_int), ("uv_pyr", C.c_int * 2), ("obs", C.c_double * 3),
                ("xyz_actkey", C.c_double * 3)]


MATCH_RESULT_DTYPE = np.dtype([("predicted", "i4"), ("textured", "i4"), ("matched", "i4"), ("n_candidates", "i4"),
                               ("index", "i4"), ("min_dist", "i4"), ("uv_pyr", "i4", 2), ("obs", "f8", 3),
                               ("xyz_actkey", "f8", 3)])
MATCH_POINT_DTYPE = np.dtype([("keyframe", "i4"), ("anchor_level", "i4"), ("xyz_anchor", "f8", 3),
                              ("anchor_obs_pyr", "f8", 2)])


class SvsFrontendParams(C.Structure):
    _fields_ = [("seed", C.c_ulonglong), ("max_reproj_error", C.c_float), ("newpoint_clearance", C.c_int),
                ("num_max_points", C.c_int), ("min_num_points", C.c_int), ("featureless_corners_thr", C.c_int),
                ("parallax_thr", C.c_float)]


def frontend_params(seed=0, max_reproj_error=2.0, newpoint_clearance=2, num_max_points=300, min_num_points=25,
                    featureless_corners_thr=2, parallax_thr=0.75):
    """svs_frontend_params; the defaults are SVS_FRONTEND_PARAMS_DEFAULT."""
    return SvsFrontendParams(int(seed), float(max_reproj_error), int(newpoint_clearance), int(num_max_points),
                             int(min_num_points), int(featureless_corners_thr), float(parallax_thr))


class SvsPointStats(C.Structure):
    _fields_ = [("num_matched_points", C.c_int * 4), ("grid2x2", C.c_int * 4), ("grid3x3", C.c_int * 9),
                ("av_track_length", C.c_double), ("num_tracked", C.c_int), ("num_new", C.c_int)]

    def as_dict(self):
        return dict(num_matched_points=list(self.num_matched_points), grid2x2=np.array(self.grid2x2[:]).reshape(2, 2),
                    grid3x3=np.array(self.grid3x3[:]).reshape(3, 3), av_track_length=self.av_track_length,
                    num_tracked=self.num_tracked, num_new=self.num_new)


# svs_tracked_point / svs_new_point
TRACKED_POINT_DTYPE = np.dtype([("index", "i4"), ("is_new", "i4"), ("anchor_level", "i4"), ("reserved", "i4"),
                                ("uvu", "f8", 3)])
NEW_POINT_DTYPE = np.dtype([("level", "i4"), ("reserved", "i4"), ("uv_pyr", "f8", 2), ("uvu_pyr", "f8", 3),
                            ("xyz", "f8", 3), ("normal", "f8", 3)])


class SvsPlaceParams(C.Structure):
    _fields_ = [("num_ransac", C.c_int), ("pixel_thr", C.c_double), ("seed", C.c_ulonglong)]


class SvsPlaceResult(C.Structure):
    _fields_ = [("best_keyframe_id", C.c_int), ("best_score", C.c_float), ("num_matches", C.c_int),
                ("num_inliers", C.c_int), ("loop_found", C.c_int), ("T_query_from_loop", C.c_double * 7),
                ("ms", C.c_float)]


class SvsLoopResult(C.Structure):
    _fields_ = [("verified", C.c_int), ("stage", C.c_int), ("n_candidates", C.c_int), ("n_matched1", C.c_int),
                ("n_matched2", C.c_int), ("n_tracks", C.c_int), ("num_left", C.c_int), ("num_right", C.c_int),
                ("num_upper", C.c_int), ("num_lower", C.c_int), ("T_align1", C.c_double * 7),
                ("T_newloop_from_oldloop", C.c_double * 7), ("T_newloop_from_w", C.c_double * 7),
                ("lm", SvsPoseStats * 2)]


REGISTER_COUNTS = ("registered", "stage", "n_direct", "n_neighborhood", "n_candidates", "n_matched1", "n_matched2", "n_tracks",
                   "n_stats", "n_neighbors", "n_committed")


class SvsRegisterResult(C.Structure):
    _fields_ = [(f, C.c_int) for f in REGISTER_COUNTS] + [
        ("T_align1", C.c_double * 7), ("T_newroot_from_oldroot", C.c_double * 7), ("T_newroot_from_w", C.c_double * 7),
        ("lm", SvsPoseStats * 2)]


# svs_register_stats
REGISTER_STATS_DTYPE = np.dtype([("vertex", np.int32), ("strength", np.int32), ("num_left", np.int32),
                                 ("num_right", np.int32), ("num_upper", np.int32), ("num_lower", np.int32),
                                 ("qualified", np.int32)])


EXPORTS = [
    "svs_ba_create", "svs_ba_destroy", "svs_last_error", "svs_ba_set_problem", "svs_ba_optimize",
    "svs_ba_get_poses", "svs_ba_get_points", "svs_ba_reset_state", "svs_optimiseInnerAndOuterWindow",
    "svs_ba_chi2", "svs_ba_reduced_system", "svs_ba_solve_reduced", "svs_device_info",
    "svs_ba_set_structure", "svs_ba_lm_begin", "svs_ba_trial_build", "svs_ba_system_buffers", "svs_ba_trial_solve",
    "svs_ba_trial_decide", "svs_ba_lm_stats",
    "svs_comm_unique_id", "svs_ba_comm_init", "svs_ba_set_problem_sharded", "svs_ba_get_points_all",
    "svs_fast_create", "svs_fast_destroy", "svs_fast_last_error", "svs_fast_grid_init", "svs_fast_set_image",
    "svs_fast_set_image_device", "svs_fast_detect", "svs_fast_detect_adaptively",
    "svs_dt_create", "svs_dt_destroy", "svs_dt_last_error", "svs_dt_set_intrinsics", "svs_dt_set_images",
    "svs_dt_set_disparity", "svs_dt_compute_point_cloud", "svs_dt_set_point_cloud", "svs_dt_get_point_cloud",
    "svs_dt_chi2", "svs_dt_jacobian_reduction", "svs_dt_track", "svs_dt_residual_image",
    "svs_matcher_create", "svs_matcher_destroy", "svs_matcher_last_error", "svs_matcher_set_keyframe",
    "svs_matcher_set_current", "svs_matcher_set_features", "svs_matcher_set_features_from_fast", "svs_match",
    "svs_prep_create", "svs_prep_destroy", "svs_prep_last_error", "svs_prep_process", "svs_prep_level",
    "svs_prep_get_u8", "svs_prep_get_f32", "svs_dt_set_images_device", "svs_dt_swap_prev_cur",
    "svs_matcher_set_pyramid_device",
    "svs_pose_create", "svs_pose_destroy", "svs_pose_last_error", "svs_calcFastMotionOnly",
    "svs_calcFastMotionOnly_matched", "svs_calcFastMotionOnly_device", "svs_pose_grad",
    "svs_dtc_create", "svs_dtc_destroy", "svs_dtc_last_error", "svs_dtc_set_prev_u8", "svs_dtc_set_cur",
    "svs_dtc_set_disparity", "svs_computeDensePointCloudCpu", "svs_dtc_get_point_cloud", "svs_dtc_set_point_cloud",
    "svs_denseTrackingCpu",
    "svs_constraints_create", "svs_constraints_destroy", "svs_constraints_last_error", "svs_computeConstraint_batch",
    "svs_map_create", "svs_map_destroy", "svs_map_last_error", "svs_map_set", "svs_map_update_poses",
    "svs_map_update_points", "svs_map_get", "svs_map_absorb", "svs_map_set_graph", "svs_map_select_window",
    "svs_map_add_keyframe", "svs_map_set_pose_graph", "svs_map_get_graph", "svs_map_add_keyframe_graph", "svs_map_add_edges",
    "svs_map_prepare_for_optimization", "svs_map_get_window_state",
    "svs_ba_set_problem_from_map", "svs_map_last_edges",
    "svs_chol6_create", "svs_chol6_destroy", "svs_chol6_last_error", "svs_chol6_init", "svs_chol6_solve",
    "svs_chol6_solve_blocks", "svs_chol6_solve_pattern",
    "svs_ba_covariance", "svs_ba_set_problem_device", "svs_ba_observation_grad", "svs_ba_window_grad",
    "svs_place_create", "svs_place_destroy", "svs_place_last_error", "svs_place_add_location", "svs_place_num_places",
    "svs_place_last_words", "svs_place_last_scores", "svs_place_last_matches", "svs_place_last_hypotheses",
    "svs_globalLoopClosure", "svs_localRegisterFrame",
    "svs_match_track", "svs_processMatchedPoints", "svs_shallWeDropNewKeyframe", "svs_addMorePoints",
    "svs_stereo_create", "svs_stereo_destroy", "svs_stereo_last_error", "svs_stereo_compute", "svs_stereo_disparity",
    "svs_stereo_get", "svs_dt_set_disparity_device", "svs_dtc_set_disparity_device", "svs_matcher_set_disparity_device",
]


def comm_unique_id():
    """128-byte NCCL rendezvous id (rank 0 creates it, the caller broadcasts it)."""
    buf = C.create_string_buffer(128)
    rc = lib().svs_comm_unique_id(buf)
    if rc != 0:
        raise SvsError(rc, "svs_comm_unique_id: NCCL not loadable")
    return buf.raw


def lib():
    """Load libsvsb200.so; raises if it was not built (no fallback)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    for prefix in ("ba", "chol6", "fast", "dt", "dtc", "prep", "matcher", "pose", "place", "map", "constraints",
                   "stereo"):
        destroy = getattr(L, f"svs_{prefix}_destroy")
        destroy.argtypes, destroy.restype = [vp], None
        last_error = getattr(L, "svs_last_error" if prefix == "ba" else f"svs_{prefix}_last_error")
        last_error.argtypes, last_error.restype = [vp], C.c_char_p
    L.svs_ba_create.argtypes = [C.POINTER(SvsBaOpts), C.POINTER(vp)]
    prob = [C.c_int, c_dp, c_up, C.c_int, c_dp, C.c_int, c_ip, c_ip, c_ip, c_dp, c_dp,
            C.c_int, c_ip, c_ip, c_dp, c_dp, C.POINTER(SvsCam)]
    L.svs_ba_set_problem.argtypes = [vp] + prob
    L.svs_ba_set_problem_device.argtypes = [vp, C.c_int, vp, vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp,
                                            C.c_int, vp, vp, vp, vp, C.POINTER(SvsCam)]
    L.svs_ba_optimize.argtypes = [vp, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.POINTER(SvsBaStats)]
    L.svs_ba_get_poses.argtypes = [vp, c_dp]
    L.svs_ba_get_points.argtypes = [vp, c_dp]
    L.svs_ba_reset_state.argtypes = [vp]
    L.svs_optimiseInnerAndOuterWindow.argtypes = [vp] + prob + [C.c_int, C.c_int, C.c_double, C.POINTER(SvsBaStats)]
    L.svs_ba_chi2.argtypes = [vp, C.c_int, C.c_double, c_dp]
    L.svs_ba_reduced_system.argtypes = [vp, C.c_int, C.c_double, C.c_double, c_dp, c_dp, c_dp]
    L.svs_ba_solve_reduced.argtypes = [vp, C.c_int, C.c_double, C.c_double, c_dp]
    L.svs_ba_covariance.argtypes = [vp, C.c_int, C.c_double, C.c_double, c_dp, C.c_int, c_ip, c_ip, c_dp, c_dp,
                                    C.POINTER(SvsBaCovStats)]
    L.svs_ba_observation_grad.argtypes = [vp, C.c_int, C.c_double, C.c_double, vp, vp, vp, vp, C.c_int,
                                          C.POINTER(SvsBaGradStats)]
    L.svs_ba_window_grad.argtypes = [vp, C.c_int, C.c_double, C.c_double, vp, vp, C.POINTER(SvsBaGradOut), C.c_int,
                                     C.POINTER(SvsBaGradStats)]
    L.svs_device_info.argtypes = [C.c_char_p, C.c_int]
    L.svs_ba_set_structure.argtypes = [vp, C.c_int, c_ip, c_ip]
    L.svs_ba_lm_begin.argtypes = [vp, C.c_double, C.c_int]
    L.svs_ba_trial_build.argtypes = [vp, C.c_int, C.c_double]
    pp = C.POINTER(C.c_void_p)
    pl = C.POINTER(C.c_longlong)
    L.svs_ba_system_buffers.argtypes = [vp, pp, pl, pp, pp, pl, pp]
    L.svs_ba_trial_solve.argtypes = [vp, C.c_int, C.c_double]
    L.svs_ba_trial_decide.argtypes = [vp, c_ip, c_ip, c_ip]
    L.svs_ba_lm_stats.argtypes = [vp, C.POINTER(SvsBaStats)]
    L.svs_comm_unique_id.argtypes = [C.c_char_p]
    L.svs_ba_comm_init.argtypes = [vp, C.c_int, C.c_int, C.c_char_p]
    L.svs_ba_set_problem_sharded.argtypes = [vp] + prob
    L.svs_ba_get_points_all.argtypes = [vp, c_dp]
    L.svs_chol6_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.svs_chol6_init.argtypes = [vp]
    L.svs_chol6_solve.argtypes = [vp, C.c_int, c_ip, c_ip, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                  C.POINTER(SvsChol6Stats)]
    L.svs_chol6_solve_blocks.argtypes = [vp, C.c_int, c_ip, c_ip, C.c_void_p, C.c_void_p, C.c_int,
                                         C.POINTER(SvsChol6InvStats)]
    L.svs_chol6_solve_pattern.argtypes = [vp, C.c_int, c_ip, c_ip, C.c_void_p, C.c_int, c_ip, c_ip, C.c_void_p, C.c_int,
                                          C.POINTER(SvsChol6InvStats)]
    L.svs_fast_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
    L.svs_fast_grid_init.argtypes = [C.c_int] * 9 + [C.POINTER(SvsFastGridParams), C.POINTER(SvsFastCell)]
    L.svs_fast_set_image.argtypes = [vp, c_up, C.c_int, C.c_int, C.c_int]
    L.svs_fast_set_image_device.argtypes = [vp, C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.svs_fast_detect.argtypes = [vp, C.POINTER(SvsFastCell), C.c_int, c_ip, C.c_int, c_ip]
    L.svs_fast_detect_adaptively.argtypes = [vp, C.POINTER(SvsFastGridParams), C.POINTER(SvsFastCell), C.c_int,
                                             c_ip, C.c_int, c_ip]
    c_fp = C.POINTER(C.c_float)
    L.svs_dt_create.argtypes = [C.c_int] * 5 + [C.POINTER(vp)]
    L.svs_dt_set_intrinsics.argtypes = [vp, C.c_int, C.c_float, C.c_float, C.c_float]
    L.svs_dt_set_images.argtypes = [vp, C.c_int, c_fp, c_fp, c_fp, c_fp, C.c_int]
    L.svs_dt_set_disparity.argtypes = [vp, c_fp, C.c_int, C.c_int, C.c_int]
    L.svs_dt_compute_point_cloud.argtypes = [vp, c_dp, C.POINTER(SvsCam)]
    L.svs_dt_set_point_cloud.argtypes = [vp, C.c_int, c_fp]
    L.svs_dt_get_point_cloud.argtypes = [vp, C.c_int, c_fp]
    L.svs_dt_chi2.argtypes = [vp, C.c_int, c_dp, c_dp]
    L.svs_dt_jacobian_reduction.argtypes = [vp, C.c_int, c_dp, c_dp, c_dp, c_dp]
    L.svs_dt_track.argtypes = [vp, c_dp, C.POINTER(SvsDtStats)]
    L.svs_dt_residual_image.argtypes = [vp, C.c_int, c_dp, c_fp]
    L.svs_prep_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
    L.svs_prep_process.argtypes = [vp, c_up, C.c_int]
    pvp = C.POINTER(C.c_void_p)
    L.svs_prep_level.argtypes = [vp, C.c_int, c_ip, c_ip, pvp, c_ip, pvp, pvp, pvp, c_ip]
    L.svs_prep_get_u8.argtypes = [vp, C.c_int, c_up]
    L.svs_prep_get_f32.argtypes = [vp, C.c_int, C.c_int, c_fp]
    L.svs_dt_set_images_device.argtypes = [vp, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    L.svs_dt_swap_prev_cur.argtypes = [vp]
    L.svs_matcher_set_pyramid_device.argtypes = [vp, C.c_int, c_dp, C.POINTER(C.c_void_p), c_ip]
    L.svs_stereo_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
    L.svs_stereo_compute.argtypes = [vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int]
    L.svs_stereo_disparity.argtypes = [vp, pvp, c_ip]
    L.svs_stereo_get.argtypes = [vp, c_fp]
    L.svs_dt_set_disparity_device.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int]
    L.svs_dtc_set_disparity_device.argtypes = [vp, vp, C.c_int]
    L.svs_matcher_set_disparity_device.argtypes = [vp, vp, C.c_int]
    L.svs_map_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.svs_map_set.argtypes = [vp, C.c_int, c_dp, C.c_int, c_ip, c_dp, c_ip, c_ip, c_dp, c_ip]
    L.svs_map_update_poses.argtypes = [vp, C.c_int, c_ip, c_dp]
    L.svs_map_update_points.argtypes = [vp, C.c_int, c_ip, c_dp]
    L.svs_map_get.argtypes = [vp, c_dp, c_dp]
    L.svs_map_absorb.argtypes = [vp, vp]
    L.svs_map_set_graph.argtypes = [vp, c_ip, c_ip, c_dp, c_dp]
    L.svs_map_select_window.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, c_ip, c_ip, c_up, C.c_int, c_ip, c_ip, C.c_int, c_ip,
                                        c_ip, c_ip, c_dp, c_dp]
    L.svs_map_add_keyframe.argtypes = [vp, C.c_int, c_dp, C.c_int, c_ip, c_dp, c_dp, c_ip, c_dp, c_ip, C.c_int, c_ip, c_dp, c_ip,
                                       c_ip, c_ip]
    L.svs_map_set_pose_graph.argtypes = [vp, c_ip, c_ip, c_ip, c_dp, c_dp]
    L.svs_map_get_graph.argtypes = [vp, C.c_int, c_ip, c_ip, c_ip, c_ip, c_dp, c_dp]
    L.svs_map_add_keyframe_graph.argtypes = [vp, C.c_int, c_dp, C.c_int, c_ip, c_dp, c_dp, c_ip, c_dp, c_ip, C.c_int, c_ip, c_dp,
                                             c_ip, C.c_int, C.c_int, C.c_int, c_ip, c_ip, c_ip, c_ip, c_ip]
    L.svs_map_add_edges.argtypes = [vp, C.c_int, c_ip, c_ip, c_ip, C.c_int, c_dp]
    L.svs_map_prepare_for_optimization.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, c_ip, C.c_int, c_ip, c_ip, c_up, C.c_int,
                                                   c_ip, c_ip, C.c_int, c_ip, c_ip, c_ip, c_dp, c_dp]
    L.svs_map_get_window_state.argtypes = [vp, C.c_int, c_ip, c_up, c_up]
    L.svs_ba_set_problem_from_map.argtypes = [vp, vp, C.c_int, c_ip, c_up, C.c_int, c_ip, C.c_int, c_ip, c_ip, c_dp, c_dp,
                                              C.POINTER(SvsCam), c_ip]
    L.svs_map_last_edges.argtypes = [vp, C.c_int, c_ip, c_ip, c_ip, c_dp, c_dp]
    L.svs_globalLoopClosure.argtypes = [vp, vp, vp, C.POINTER(SvsCam), C.c_int, C.c_int, C.c_int, c_dp, C.c_int, c_ip, c_ip,
                                        C.POINTER(SvsLoopResult), C.c_int, c_ip, c_dp, c_ip]
    L.svs_localRegisterFrame.argtypes = [vp, vp, vp, C.POINTER(SvsCam), C.c_int, C.c_int, C.c_int, c_ip, c_ip,
                                         C.POINTER(SvsRegisterResult), C.c_int, vp, C.c_int, c_ip, c_dp, c_ip, c_ip]
    L.svs_constraints_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.svs_computeConstraint_batch.argtypes = [vp, C.c_int, c_dp, c_ip, c_ip, C.c_int, c_ip, c_dp, C.c_int, c_ip, c_ip,
                                              c_dp, c_dp, c_ip]
    L.svs_dtc_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
    L.svs_dtc_set_prev_u8.argtypes = [vp, C.c_int, C.c_void_p, C.c_int, C.c_int]
    L.svs_dtc_set_cur.argtypes = [vp, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.svs_dtc_set_disparity.argtypes = [vp, c_fp, C.c_int]
    L.svs_computeDensePointCloudCpu.argtypes = [vp, c_dp, C.POINTER(SvsCam)]
    L.svs_dtc_get_point_cloud.argtypes = [vp, C.c_int, c_fp]
    L.svs_dtc_set_point_cloud.argtypes = [vp, C.c_int, c_fp]
    L.svs_denseTrackingCpu.argtypes = [vp, C.POINTER(SvsCam), c_dp, C.POINTER(SvsDtStats)]
    L.svs_pose_create.argtypes = [C.c_int, C.c_int, C.POINTER(vp)]
    L.svs_calcFastMotionOnly.argtypes = [vp, C.c_int, c_ip, c_dp, C.c_int, c_dp, C.POINTER(SvsCam),
                                         C.POINTER(SvsPoseParams), c_dp, C.POINTER(SvsPoseStats)]
    L.svs_calcFastMotionOnly_matched.argtypes = [vp, vp, C.POINTER(SvsCam), C.POINTER(SvsPoseParams), c_dp,
                                                 C.POINTER(SvsPoseStats)]
    L.svs_calcFastMotionOnly_device.argtypes = [vp, C.c_int, vp, vp, C.c_int, vp, C.POINTER(SvsCam),
                                                C.POINTER(SvsPoseParams), c_dp, C.POINTER(SvsPoseStats)]
    L.svs_pose_grad.argtypes = [vp, C.c_double, vp, vp, vp, vp, C.c_int, C.POINTER(SvsPoseGradStats)]
    ucpp = C.POINTER(C.POINTER(C.c_ubyte))
    L.svs_matcher_create.argtypes = [C.c_int, C.c_int, C.POINTER(SvsMatchLevel), C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
    L.svs_matcher_set_keyframe.argtypes = [vp, C.c_int, c_dp, ucpp, c_ip]
    L.svs_matcher_set_current.argtypes = [vp, ucpp, c_ip, c_fp, C.c_int]
    L.svs_matcher_set_features.argtypes = [vp, C.c_int, c_ip, c_ip, C.c_int]
    L.svs_matcher_set_features_from_fast.argtypes = [vp, C.c_int, vp]
    L.svs_match.argtypes = [vp, c_dp, c_dp, C.POINTER(SvsMatchPoint), C.c_int, C.c_int, C.c_int, C.c_int,
                            C.POINTER(SvsMatchResult)]
    L.svs_match_track.argtypes = [vp, c_dp, c_dp, C.POINTER(SvsMatchPoint), C.c_int, C.c_int, c_ip, C.c_int, C.c_int,
                                  C.c_int, C.c_int, C.POINTER(SvsMatchResult), c_ip, c_ip]
    L.svs_processMatchedPoints.argtypes = [vp, c_dp, C.POINTER(SvsCam), C.c_int, C.POINTER(SvsFrontendParams), vp,
                                           C.POINTER(SvsPointStats), c_ip, c_ip]
    L.svs_shallWeDropNewKeyframe.argtypes = [C.POINTER(SvsPointStats), c_dp, C.POINTER(SvsFrontendParams)]
    L.svs_addMorePoints.argtypes = [vp, C.c_int, c_dp, C.POINTER(SvsCam), C.c_int, C.POINTER(SvsFrontendParams), vp, vp,
                                    C.c_int, c_ip]
    L.svs_place_create.argtypes = [C.c_int, C.c_int, c_fp, C.POINTER(SvsCam), C.POINTER(vp)]
    L.svs_place_add_location.argtypes = [vp, C.c_int, C.c_int, c_fp, c_dp, C.c_int, C.c_int, c_ip,
                                         C.POINTER(SvsPlaceParams), C.POINTER(SvsPlaceResult), c_ip, c_ip]
    L.svs_place_num_places.argtypes = [vp]
    L.svs_place_last_words.argtypes = [vp, c_ip]
    L.svs_place_last_scores.argtypes = [vp, C.c_int, c_ip, c_fp]
    L.svs_place_last_matches.argtypes = [vp, c_ip, c_fp]
    L.svs_place_last_hypotheses.argtypes = [vp, C.c_int, c_ip, c_ip, c_ip]
    _LIB = L
    return L


def device_info() -> str:
    buf = C.create_string_buffer(256)
    rc = lib().svs_device_info(buf, 256)
    if rc != 0:
        raise RuntimeError(f"svs_device_info: {buf.value.decode()} (rc={rc})")
    return buf.value.decode()


def _dp(a):
    return a.ctypes.data_as(c_dp)


def _ip(a):
    return a.ctypes.data_as(c_ip)


def _is_torch_tensor(a):
    t = type(a)
    return t.__module__.startswith("torch") and t.__name__ == "Tensor"


class SvsError(RuntimeError):
    def __init__(self, rc, msg):
        super().__init__(f"svs error {rc}: {msg}")
        self.rc = rc


class _Handle:
    """One opaque handle of the C ABI.  A subclass names its destroy and last-error functions; close() (or the
    garbage collector) destroys the handle."""
    _destroy = _last_error = None
    _h = None

    def _open(self, create, *args, why="no CUDA device? there is no CPU fallback"):
        self._h = C.c_void_p()
        rc = getattr(lib(), create)(*args, C.byref(self._h))
        if rc != 0:
            raise SvsError(rc, f"{create} failed ({why})")

    def close(self):
        if self._h:
            getattr(lib(), self._destroy)(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _error(self, rc):
        return SvsError(rc, getattr(lib(), self._last_error)(self._h).decode())

    def _ck(self, rc):
        if rc != 0:
            raise self._error(rc)


class BundleAdjuster(_Handle):
    """Thin host-side mirror of SlamGraph::optimize (reference slam_graph.cpp:319-355)."""

    _destroy, _last_error = "svs_ba_destroy", "svs_last_error"

    def __init__(self, device: int = -1, flags: int = 0):
        o = SvsBaOpts(device, flags)
        self._open("svs_ba_create", C.byref(o))
        self._keep = None
        self.P = self.L = self.E = self.C = 0

    @staticmethod
    def _arrays(pb):
        return dict(
            pose_qt=np.ascontiguousarray(pb.pose_qt, np.float64), fixed=np.ascontiguousarray(pb.fixed, np.uint8),
            psi=np.ascontiguousarray(pb.psi, np.float64),
            e_point=np.ascontiguousarray(pb.e_point, np.int32), e_pose=np.ascontiguousarray(pb.e_pose, np.int32),
            e_anchor=np.ascontiguousarray(pb.e_anchor, np.int32),
            e_obs=np.ascontiguousarray(pb.e_obs, np.float64), e_info=np.ascontiguousarray(pb.e_info, np.float64),
            c_i=np.ascontiguousarray(pb.c_i, np.int32), c_j=np.ascontiguousarray(pb.c_j, np.int32),
            c_T=np.ascontiguousarray(pb.c_T, np.float64), c_Lambda=np.ascontiguousarray(pb.c_Lambda, np.float64))

    @staticmethod
    def _prob_args(pb, k):
        cam = SvsCam(float(pb.cam[0]), float(pb.cam[1]), float(pb.cam[2]), float(pb.cam[3]))
        return [pb.P, _dp(k["pose_qt"]), k["fixed"].ctypes.data_as(c_up), pb.L, _dp(k["psi"]),
                pb.E, _ip(k["e_point"]), _ip(k["e_pose"]), _ip(k["e_anchor"]), _dp(k["e_obs"]), _dp(k["e_info"]),
                pb.C, _ip(k["c_i"]), _ip(k["c_j"]), _dp(k["c_T"]), _dp(k["c_Lambda"]), C.byref(cam)], cam

    _DEVICE_ARRAYS = (("pose_qt", "float64"), ("fixed", "uint8"), ("psi", "float64"), ("e_point", "int32"),
                      ("e_pose", "int32"), ("e_anchor", "int32"), ("e_obs", "float64"), ("e_info", "float64"),
                      ("c_i", "int32"), ("c_j", "int32"), ("c_T", "float64"), ("c_Lambda", "float64"))

    def set_problem(self, pb):
        """Load a window.  Its arrays are numpy arrays, or CUDA torch tensors on the handle's device (int32 indices,
        uint8 fixed flags or None, float64 numbers): then the window never passes through the host and its structure
        is analysed on the device (svs_ba_set_problem_device).  The current torch stream is synchronised first."""
        if any(_is_torch_tensor(getattr(pb, name)) for name, _ in self._DEVICE_ARRAYS):
            self._set_problem_device(pb)
        else:
            k = self._arrays(pb)
            args, cam = self._prob_args(pb, k)
            self._ck(lib().svs_ba_set_problem(self._h, *args))
        self.P, self.L, self.E, self.C = pb.P, pb.L, pb.E, pb.C

    def _set_problem_device(self, pb):
        import torch
        ptr, keep, dev = {}, [], None
        for name, dtype in self._DEVICE_ARRAYS:
            t = getattr(pb, name)
            if name == "fixed" and t is None:
                ptr[name] = None
                continue
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == getattr(torch, dtype)):
                raise TypeError(f"{name}: a CUDA {dtype} tensor (all arrays of a device problem are)")
            if dev is not None and t.device != dev:
                raise ValueError(f"{name}: on {t.device}, the other arrays on {dev}")
            dev = t.device
            t = t.contiguous()
            keep.append(t)
            ptr[name] = t.data_ptr() if t.numel() else None
        cam = SvsCam(float(pb.cam[0]), float(pb.cam[1]), float(pb.cam[2]), float(pb.cam[3]))
        torch.cuda.current_stream(dev).synchronize()   # the handle reads the arrays on its own stream
        p = ptr
        self._ck(lib().svs_ba_set_problem_device(
            self._h, int(pb.P), p["pose_qt"], p["fixed"], int(pb.L), p["psi"], int(pb.E), p["e_point"], p["e_pose"],
            p["e_anchor"], p["e_obs"], p["e_info"], int(pb.C), p["c_i"], p["c_j"], p["c_T"], p["c_Lambda"],
            C.byref(cam)))

    def optimize(self, num_iters, robust=True, huber_delta=1.0, lambda_init=50.0, max_trials=5):
        st = SvsBaStats()
        it = lib().svs_ba_optimize(self._h, int(num_iters), int(robust), float(huber_delta), float(lambda_init),
                                   int(max_trials), C.byref(st))
        if it <= -100:
            self._ck(it + 100)
        return it, st.as_dict()

    def poses(self):
        out = np.zeros((self.P, 7))
        self._ck(lib().svs_ba_get_poses(self._h, _dp(out)))
        return out

    def points(self):
        out = np.zeros((self.L, 3))
        self._ck(lib().svs_ba_get_points(self._h, _dp(out)))
        return out

    def reset_state(self):
        self._ck(lib().svs_ba_reset_state(self._h))

    def chi2(self, robust=True, huber_delta=1.0):
        v = C.c_double()
        self._ck(lib().svs_ba_chi2(self._h, int(robust), float(huber_delta), C.byref(v)))
        return v.value

    def reduced_system(self, robust=True, huber_delta=1.0, lam=50.0):
        n = 6 * self.P
        S, bs = np.zeros((n, n)), np.zeros(n)
        chi = C.c_double()
        self._ck(lib().svs_ba_reduced_system(self._h, int(robust), float(huber_delta), float(lam), _dp(S), _dp(bs),
                                             C.byref(chi)))
        return S, bs, chi.value

    def solve_reduced(self, robust=True, huber_delta=1.0, lam=50.0):
        x = np.zeros(6 * self.P)
        rc = lib().svs_ba_solve_reduced(self._h, int(robust), float(huber_delta), float(lam), _dp(x))
        if rc < 0:
            self._ck(rc)
        return x, rc

    def covariance(self, robust=True, huber_delta=1.0, lam=0.0, pairs=()):
        """Marginal covariances at the accepted state (svs_ba_covariance): blocks of (H + lam I)^-1 over the free
        variables, zero for fixed poses.  Returns (pose_cov [P,6,6], pair_cov [n,6,6] with pair_cov[k] =
        Cov(x_i, x_j) for pairs[k] = (i, j), point_cov [L,3,3] in psi, rc, stats); rc = 1: not positive definite
        (outputs zeroed)."""
        pr = np.ascontiguousarray(np.asarray(pairs, np.int32).reshape(-1, 2))
        pi, pj = np.ascontiguousarray(pr[:, 0]), np.ascontiguousarray(pr[:, 1])
        n = len(pr)
        pose, pair, point = np.zeros((self.P, 6, 6)), np.zeros((n, 6, 6)), np.zeros((self.L, 3, 3))
        st = SvsBaCovStats()
        rc = lib().svs_ba_covariance(self._h, int(robust), float(huber_delta), float(lam), _dp(pose), n,
                                     _ip(pi) if n else None, _ip(pj) if n else None, _dp(pair) if n else None,
                                     _dp(point), C.byref(st))
        if rc < 0:
            self._ck(rc)
        return pose, pair, point, rc, st.as_dict()

    def observation_grad(self, dL_dpose=None, dL_dpsi=None, robust=True, huber_delta=1.0, lam=0.0):
        """dL/d(observations, weights) of the optimised window at the accepted state (svs_ba_observation_grad) from
        dL_dpose [P,6] (upsilon, omega) and dL_dpsi [L,3] (None = 0).  Returns (dL_dobs [E,3], dL_dinfo [E,3] in the
        caller's edge order, rc, stats); rc = 1: not positive definite (outputs zeroed).  Numpy arrays in, numpy out;
        CUDA float64 tensors on the handle's device in, tensors out (the current torch stream is synchronised first)."""
        st = SvsBaGradStats()
        if _is_torch_tensor(dL_dpose) or _is_torch_tensor(dL_dpsi):
            import torch
            ins = [t for t in (dL_dpose, dL_dpsi) if t is not None]
            dev = ins[0].device
            for t in ins:
                if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float64 and t.device == dev):
                    raise TypeError("dL_dpose / dL_dpsi: CUDA float64 tensors on one device (or None)")
            gp = None if dL_dpose is None else dL_dpose.detach().reshape(self.P, 6).contiguous()
            gl = None if dL_dpsi is None else dL_dpsi.detach().reshape(self.L, 3).contiguous()
            dobs = torch.empty((self.E, 3), dtype=torch.float64, device=dev)
            dinfo = torch.empty((self.E, 3), dtype=torch.float64, device=dev)
            torch.cuda.current_stream(dev).synchronize()   # the handle reads the arrays on its own stream
            ptr = lambda t: t.data_ptr() if t is not None and t.numel() else None
            rc = lib().svs_ba_observation_grad(self._h, int(robust), float(huber_delta), float(lam), ptr(gp), ptr(gl),
                                               ptr(dobs), ptr(dinfo), 1, C.byref(st))
        else:
            gp = None if dL_dpose is None else np.ascontiguousarray(np.asarray(dL_dpose, np.float64).reshape(self.P, 6))
            gl = None if dL_dpsi is None else np.ascontiguousarray(np.asarray(dL_dpsi, np.float64).reshape(self.L, 3))
            dobs, dinfo = np.zeros((self.E, 3)), np.zeros((self.E, 3))
            ptr = lambda a: a.ctypes.data if a is not None and a.size else None
            rc = lib().svs_ba_observation_grad(self._h, int(robust), float(huber_delta), float(lam), ptr(gp), ptr(gl),
                                               ptr(dobs), ptr(dinfo), 0, C.byref(st))
        if rc < 0:
            self._ck(rc)
        return dobs, dinfo, rc, st.as_dict()

    # outputs of window_grad: name -> (svs_ba_grad_out member, trailing shape)
    _GRAD_OUT = {"obs": ("dL_dobs", (3,)), "info": ("dL_dinfo", (3,)), "cT": ("dL_dcT", (6,)),
                 "cLambda": ("dL_dcLambda", (36,)), "cam": ("dL_dcam", ())}

    def window_grad(self, dL_dpose=None, dL_dpsi=None, robust=True, huber_delta=1.0, lam=0.0,
                    want=("obs", "info", "cT", "cLambda", "cam")):
        """svs_ba_window_grad: observation_grad extended to the pose-pose constraints and the camera, from one adjoint
        solve.  `want` names the outputs to compute, any of "obs" / "info" [E,3] (caller's edge order), "cT" [C,6]
        (tangent (upsilon, omega) of T_ji <- exp(d) T_ji), "cLambda" [C,36] (row-major, symmetric), "cam" [4]
        (f, px, py, b); the others are neither computed nor written.  Returns (dict name -> array for the names in
        `want`, rc, stats); rc = 1: not positive definite (outputs zeroed).  Numpy arrays in, numpy out; CUDA float64
        tensors on the handle's device in, tensors out (the current torch stream is synchronised first)."""
        bad = [w for w in want if w not in self._GRAD_OUT]
        if bad:
            raise ValueError(f"want: unknown outputs {bad} (choose from {list(self._GRAD_OUT)})")
        rows = {"obs": self.E, "info": self.E, "cT": self.C, "cLambda": self.C}
        shape = lambda w: (4,) if w == "cam" else (rows[w],) + self._GRAD_OUT[w][1]
        st, out = SvsBaGradStats(), SvsBaGradOut()
        if _is_torch_tensor(dL_dpose) or _is_torch_tensor(dL_dpsi):
            import torch
            ins = [t for t in (dL_dpose, dL_dpsi) if t is not None]
            dev = ins[0].device
            for t in ins:
                if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float64 and t.device == dev):
                    raise TypeError("dL_dpose / dL_dpsi: CUDA float64 tensors on one device (or None)")
            gp = None if dL_dpose is None else dL_dpose.detach().reshape(self.P, 6).contiguous()
            gl = None if dL_dpsi is None else dL_dpsi.detach().reshape(self.L, 3).contiguous()
            res = {w: torch.empty(shape(w), dtype=torch.float64, device=dev) for w in want}
            torch.cuda.current_stream(dev).synchronize()   # the handle reads the arrays on its own stream
            ptr = lambda t: t.data_ptr() if t is not None and t.numel() else None
            on_device = 1
        else:
            gp = None if dL_dpose is None else np.ascontiguousarray(np.asarray(dL_dpose, np.float64).reshape(self.P, 6))
            gl = None if dL_dpsi is None else np.ascontiguousarray(np.asarray(dL_dpsi, np.float64).reshape(self.L, 3))
            res = {w: np.zeros(shape(w)) for w in want}
            ptr = lambda a: a.ctypes.data if a is not None and a.size else None
            on_device = 0
        for w, a in res.items():
            setattr(out, self._GRAD_OUT[w][0], ptr(a))
        rc = lib().svs_ba_window_grad(self._h, int(robust), float(huber_delta), float(lam), ptr(gp), ptr(gl),
                                      C.byref(out), on_device, C.byref(st))
        if rc < 0:
            self._ck(rc)
        return res, rc, st.as_dict()

    # ---- stepwise trial API (window split by landmarks across ranks, SURVEY.md 8e)
    def set_structure(self, pairs):
        pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
        pi, pj = np.ascontiguousarray(pairs[:, 0]), np.ascontiguousarray(pairs[:, 1])
        self._ck(lib().svs_ba_set_structure(self._h, len(pairs), _ip(pi), _ip(pj)))

    def lm_begin(self, lambda_init=50.0, max_trials=5):
        self._ck(lib().svs_ba_lm_begin(self._h, float(lambda_init), int(max_trials)))

    def trial_build(self, robust=True, huber_delta=1.0):
        self._ck(lib().svs_ba_trial_build(self._h, int(robust), float(huber_delta)))

    def system_buffers(self):
        """(ptr_S, nS, ptr_bp, ptr_bc, nb, ptr_totals): raw device pointers for the caller's collective."""
        S, bp, bc, tot = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        nS, nb = C.c_longlong(), C.c_longlong()
        self._ck(lib().svs_ba_system_buffers(self._h, C.byref(S), C.byref(nS), C.byref(bp), C.byref(bc), C.byref(nb),
                                             C.byref(tot)))
        return S.value, nS.value, bp.value, bc.value, nb.value, tot.value

    def trial_solve(self, robust=True, huber_delta=1.0):
        self._ck(lib().svs_ba_trial_solve(self._h, int(robust), float(huber_delta)))

    def trial_decide(self):
        a, s, i = C.c_int(), C.c_int(), C.c_int()
        self._ck(lib().svs_ba_trial_decide(self._h, C.byref(a), C.byref(s), C.byref(i)))
        return a.value, s.value, i.value

    # ---- one window sharded by landmarks across GPUs, driven inside the library (NCCL on the handle's stream)
    def comm_init(self, nranks, rank, unique_id):
        """unique_id: the 128 bytes rank 0 got from `comm_unique_id()`, broadcast by the caller."""
        self._ck(lib().svs_ba_comm_init(self._h, int(nranks), int(rank), bytes(unique_id)))

    def set_problem_sharded(self, pb):
        """Every rank passes the WHOLE window; the library keeps landmarks l % nranks == rank."""
        k = self._arrays(pb)
        args, cam = self._prob_args(pb, k)
        self._ck(lib().svs_ba_set_problem_sharded(self._h, *args))
        self.P, self.L, self.E, self.C = pb.P, pb.L, pb.E, pb.C

    def points_all(self):
        out = np.zeros((self.L, 3))
        self._ck(lib().svs_ba_get_points_all(self._h, _dp(out)))
        return out

    def lm_stats(self):
        st = SvsBaStats()
        self._ck(lib().svs_ba_lm_stats(self._h, C.byref(st)))
        return st.as_dict()

    def optimise_inner_and_outer_window(self, pb, num_iters, robust=True, huber_delta=1.0):
        """SlamGraph::optimize in one call from host buffers; returns (iters, poses, psi, stats)."""
        k = self._arrays(pb)
        k["pose_qt"] = k["pose_qt"].copy()
        k["psi"] = k["psi"].copy()
        args, cam = self._prob_args(pb, k)
        st = SvsBaStats()
        it = lib().svs_optimiseInnerAndOuterWindow(self._h, *args, int(num_iters), int(robust), float(huber_delta),
                                                   C.byref(st))
        if it <= -100:
            self._ck(it + 100)
        self.P, self.L, self.E, self.C = pb.P, pb.L, pb.E, pb.C
        return it, k["pose_qt"], k["psi"], st.as_dict()


class BlockCholesky6(_Handle):
    """g2o's LinearSolver<Matrix6d>::solve(A, x, b) on the device (svs_chol6_*): A is the upper triangle of a
    symmetric positive-definite matrix in block CCS -- col_ptr [P+1], row_idx [nnzb] (ascending, row <= column,
    every column ends in its diagonal block), blocks [nnzb][36] with each block column-major (Eigen's
    Matrix6d::data(); from numpy, B.ravel(order="F")) -- and b has 6P entries.  No damping is added."""

    _destroy, _last_error = "svs_chol6_destroy", "svs_chol6_last_error"

    def __init__(self, device: int = -1):
        self._open("svs_chol6_create", int(device))

    def init(self):
        """LinearSolver::init(): forget the cached symbolic analysis."""
        self._ck(lib().svs_chol6_init(self._h))

    def solve(self, col_ptr, row_idx, blocks, b):
        """Returns (x, status, stats): status 0 = solved, 1 = not positive definite (x is zero).  blocks and b are
        numpy arrays (x comes back as numpy) or CUDA float64 torch tensors on the handle's device (x comes back as a
        tensor there); col_ptr and row_idx are host integer arrays.  Raises SvsError for a malformed input."""
        col_ptr = np.ascontiguousarray(col_ptr, np.int32)
        row_idx = np.ascontiguousarray(row_idx, np.int32)
        P = len(col_ptr) - 1
        st = SvsChol6Stats()
        if isinstance(blocks, np.ndarray) or isinstance(b, np.ndarray):
            blocks = np.ascontiguousarray(blocks, np.float64)
            b = np.ascontiguousarray(b, np.float64)
            x = np.zeros(max(6 * P, 0))
            args = (blocks.ctypes.data, b.ctypes.data, x.ctypes.data, 0)
        else:
            import torch
            for name, t in (("blocks", blocks), ("b", b)):
                if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float64):
                    raise TypeError(f"{name}: a numpy array or a CUDA float64 tensor")
            blocks, b = blocks.contiguous(), b.contiguous()
            x = torch.zeros(max(6 * P, 0), dtype=torch.float64, device=b.device)
            torch.cuda.current_stream(b.device).synchronize()   # the handle works on its own stream
            args = (blocks.data_ptr(), b.data_ptr(), x.data_ptr(), 1)
        rc = lib().svs_chol6_solve(self._h, P, _ip(col_ptr), _ip(row_idx), C.c_void_p(args[0]), C.c_void_p(args[1]),
                                   C.c_void_p(args[2]), args[3], C.byref(st))
        if rc < 0:
            self._ck(rc)
        return x, rc, st.as_dict()

    def _inverse(self, col_ptr, row_idx, blocks, n, call):
        """Shared by solve_blocks / solve_pattern: n output blocks, host or device like `blocks`; call(P, cp, ri,
        blocks_ptr, out_ptr, on_device, stats) runs the C entry point."""
        col_ptr = np.ascontiguousarray(col_ptr, np.int32)
        row_idx = np.ascontiguousarray(row_idx, np.int32)
        P = len(col_ptr) - 1
        st = SvsChol6InvStats()
        if isinstance(blocks, np.ndarray):
            blocks = np.ascontiguousarray(blocks, np.float64)
            out = np.zeros((n, 36))
            args = (blocks.ctypes.data, out.ctypes.data, 0)
        else:
            import torch
            if not (isinstance(blocks, torch.Tensor) and blocks.is_cuda and blocks.dtype == torch.float64):
                raise TypeError("blocks: a numpy array or a CUDA float64 tensor")
            blocks = blocks.contiguous()
            out = torch.zeros((n, 36), dtype=torch.float64, device=blocks.device)
            torch.cuda.current_stream(blocks.device).synchronize()   # the handle works on its own stream
            args = (blocks.data_ptr(), out.data_ptr(), 1)
        rc = call(P, _ip(col_ptr), _ip(row_idx), C.c_void_p(args[0]), C.c_void_p(args[1]), args[2], C.byref(st))
        if rc < 0:
            self._ck(rc)
        # column-major blocks -> ordinary 6x6 matrices
        return out.reshape(n, 6, 6).swapaxes(1, 2), rc, st.as_dict()

    def solve_blocks(self, col_ptr, row_idx, blocks):
        """LinearSolver::solveBlocks: returns (inv_diag [P, 6, 6], status, stats), the diagonal blocks of A^-1;
        status 1 = not positive definite (all zero).  Inputs as for solve()."""
        P = max(len(col_ptr) - 1, 0)
        return self._inverse(col_ptr, row_idx, blocks, P, lambda *a: lib().svs_chol6_solve_blocks(self._h, *a))

    def solve_pattern(self, col_ptr, row_idx, blocks, pairs):
        """LinearSolver::solvePattern: returns (out [n, 6, 6], status, stats) with out[k] = block (r, c) of A^-1 for
        pairs[k] = (r, c), in any order; status 1 = not positive definite (all zero).  Inputs as for solve()."""
        pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
        r = np.ascontiguousarray(pairs[:, 0], np.int32)
        c = np.ascontiguousarray(pairs[:, 1], np.int32)
        n = len(pairs)
        return self._inverse(col_ptr, row_idx, blocks, n,
                             lambda P, cp, ri, bl, out, dev, st: lib().svs_chol6_solve_pattern(
                                 self._h, P, cp, ri, bl, n, _ip(r), _ip(c), out, dev, st))


class FastGrid(_Handle):
    """Host-side mirror of ScaViSLAM's FastGrid (reference fast_grid.h:30-64): same constructor
    arguments, detect / detectAdaptively on the GPU through the C ABI.  Keypoints come back as
    (xy[n,2] int32, cell_off[ncells+1]); the quadtree content of keypoint i in cell c is
    i - cell_off[c]."""

    _destroy, _last_error = "svs_fast_destroy", "svs_fast_last_error"

    def __init__(self, img_w, img_h, num_features_per_cell, boundary_per_cell, fast_thr, grid_w, grid_h,
                 fast_min=10, fast_max=40, device=-1, max_keypoints=200000):
        self._open("svs_fast_create", device, img_w, img_h, max_keypoints)
        self.params = SvsFastGridParams()
        self.cells = (SvsFastCell * (grid_w * grid_h))()
        rc = lib().svs_fast_grid_init(img_w, img_h, num_features_per_cell, boundary_per_cell, fast_thr, grid_w,
                                      grid_h, fast_min, fast_max, C.byref(self.params), self.cells)
        if rc != 0:
            raise SvsError(rc, "svs_fast_grid_init")
        self.max_kp = max_keypoints
        self.ncells = grid_w * grid_h

    def set_image(self, img):
        img = np.ascontiguousarray(img, np.uint8)
        self._ck(lib().svs_fast_set_image(self._h, img.ctypes.data_as(c_up), img.strides[0], img.shape[1], img.shape[0]))

    def set_image_device(self, ptr, pitch, w, h):
        self._ck(lib().svs_fast_set_image_device(self._h, C.c_void_p(ptr), pitch, w, h))

    def cell_list(self):
        return [(c.u0, c.u1, c.v0, c.v1, c.thr) for c in self.cells]

    def detect(self, cells=None):
        """FastGrid::detect(img, cell_grid2d, qt) with static per-cell thresholds."""
        if cells is None:
            arr, n = self.cells, self.ncells
        else:
            n = len(cells)
            arr = (SvsFastCell * n)(*[SvsFastCell(*c) for c in cells])
        out = np.zeros((self.max_kp, 2), np.int32)
        off = np.zeros(n + 1, np.int32)
        tot = lib().svs_fast_detect(self._h, arr, n, _ip(out), self.max_kp, _ip(off))
        if tot < 0:
            self._ck(tot)
        return out[:min(tot, self.max_kp)].copy(), off

    def detect_adaptively(self, trials):
        """FastGrid::detectAdaptively(img, trials, qt); updates the per-cell thresholds in place."""
        out = np.zeros((self.max_kp, 2), np.int32)
        off = np.zeros(self.ncells + 1, np.int32)
        tot = lib().svs_fast_detect_adaptively(self._h, C.byref(self.params), self.cells, int(trials), _ip(out),
                                               self.max_kp, _ip(off))
        if tot < 0:
            self._ck(tot)
        return out[:min(tot, self.max_kp)].copy(), off


class DenseTracker(_Handle):
    """Host-side mirror of DenseTracker / GpuTracker (reference dense_tracking.h:40-96,
    gpu/dense_tracking.cuh:276-342) on top of the C ABI."""

    _destroy, _last_error = "svs_dt_destroy", "svs_dt_last_error"

    def __init__(self, w0, h0, nlevels=3, flags=0, device=-1):
        self._open("svs_dt_create", device, w0, h0, nlevels, flags)
        self.w0, self.h0, self.nlevels = w0, h0, nlevels

    @staticmethod
    def _fp(a):
        return None if a is None else a.ctypes.data_as(C.POINTER(C.c_float))

    def set_intrinsics(self, level, f, px, py):
        self._ck(lib().svs_dt_set_intrinsics(self._h, level, f, px, py))

    def set_images(self, level, prev=None, cur=None, dx=None, dy=None):
        """Level images as 2-D float32 arrays of at least (h0 >> level, w0 >> level); the tracker reads that top-left
        window with each array's own row stride (a pyramid that rounds its sizes up, like cv2.pyrDown, is wider)."""
        w, h = self.w0 >> level, self.h0 >> level
        for k, a in enumerate((prev, cur, dx, dy)):
            if a is None:
                continue
            a = np.ascontiguousarray(a, np.float32)
            if a.ndim != 2 or a.shape[0] < h or a.shape[1] < w:
                raise SvsError(-1, f"level {level} image of shape {a.shape} is smaller than ({h}, {w})")
            planes = [None] * 4
            planes[k] = self._fp(a)
            self._ck(lib().svs_dt_set_images(self._h, level, *planes, a.shape[1]))

    def set_images_device(self, level, prev=None, cur=None, dx=None, dy=None, stride=0):
        self._ck(lib().svs_dt_set_images_device(self._h, level, prev, cur, dx, dy, stride))

    def swap_prev_cur(self):
        self._ck(lib().svs_dt_swap_prev_cur(self._h))

    def set_disparity(self, disp):
        d = np.ascontiguousarray(disp, np.float32)
        self._ck(lib().svs_dt_set_disparity(self._h, self._fp(d), d.shape[1], d.shape[1], d.shape[0]))

    def set_disparity_device(self, ptr, stride, w=None, h=None):
        """The level-0 map from device memory, e.g. StereoMatcher.device_disparity(); (w, h) default to the frame's."""
        self._ck(lib().svs_dt_set_disparity_device(self._h, ptr, stride, self.w0 if w is None else w,
                                                   self.h0 if h is None else h))

    def compute_point_cloud(self, T, cams):
        arr = (SvsCam * len(cams))(*[SvsCam(*map(float, c)) for c in cams])
        T = np.ascontiguousarray(T, np.float64)
        self._ck(lib().svs_dt_compute_point_cloud(self._h, _dp(T), arr))

    def set_point_cloud(self, level, cloud):
        c = np.ascontiguousarray(cloud, np.float32)
        self._ck(lib().svs_dt_set_point_cloud(self._h, level, self._fp(c)))

    def get_point_cloud(self, level):
        out = np.zeros((self.h0 >> level, self.w0 >> level, 4), np.float32)
        self._ck(lib().svs_dt_get_point_cloud(self._h, level, self._fp(out)))
        return out

    def chi2(self, level, T):
        T = np.ascontiguousarray(T, np.float64)
        v = C.c_double()
        self._ck(lib().svs_dt_chi2(self._h, level, _dp(T), C.byref(v)))
        return v.value

    def jacobian_reduction(self, level, T):
        T = np.ascontiguousarray(T, np.float64)
        H, b, v = np.zeros(21), np.zeros(6), C.c_double()
        self._ck(lib().svs_dt_jacobian_reduction(self._h, level, _dp(T), _dp(H), _dp(b), C.byref(v)))
        return H, b, v.value

    def residual_image(self, level, T):
        """GpuTracker::residualImage: (h, w, 4) float32."""
        T = np.ascontiguousarray(T, np.float64)
        out = np.zeros((self.h0 >> level, self.w0 >> level, 4), np.float32)
        self._ck(lib().svs_dt_residual_image(self._h, level, _dp(T), self._fp(out)))
        return out

    def track(self, T):
        T = np.ascontiguousarray(T, np.float64).copy()
        st = SvsDtStats()
        self._ck(lib().svs_dt_track(self._h, _dp(T), C.byref(st)))
        return T, dict(chi2=list(st.chi2[:self.nlevels]), passes=list(st.passes[:self.nlevels]),
                       launches=st.launches, ms_total=st.ms_total)


class GuidedMatcher(_Handle):
    """Host-side mirror of GuidedMatcher<StereoCamera> (reference matcher.hpp:62-186)."""

    _destroy, _last_error = "svs_matcher_destroy", "svs_matcher_last_error"

    def __init__(self, levels, max_keyframes=8, max_points=8192, max_keypoints=65536, device=-1):
        """levels: list of (w, h, f, px, py) per pyramid level (cam_vec)."""
        arr = (SvsMatchLevel * len(levels))(*[SvsMatchLevel(int(w), int(h), float(f), float(px), float(py))
                                              for (w, h, f, px, py) in levels])
        self._open("svs_matcher_create", device, len(levels), arr, max_keyframes, max_points, max_keypoints)
        self.nlevels = len(levels)
        self.max_points = max_points

    def _pyr_args(self, pyr):
        ims = [np.ascontiguousarray(p, np.uint8) for p in pyr]
        ptrs = (C.POINTER(C.c_ubyte) * len(ims))(*[im.ctypes.data_as(c_up) for im in ims])
        pitch = np.array([im.strides[0] for im in ims], np.int32)
        return ims, ptrs, pitch

    def set_keyframe(self, slot, T_me_from_w, pyr):
        ims, ptrs, pitch = self._pyr_args(pyr)
        T = np.ascontiguousarray(T_me_from_w, np.float64)
        self._ck(lib().svs_matcher_set_keyframe(self._h, slot, _dp(T), ptrs, _ip(pitch)))

    def set_current(self, pyr, disp=None):
        ims, ptrs, pitch = self._pyr_args(pyr)
        d = None if disp is None else np.ascontiguousarray(disp, np.float32)
        self._ck(lib().svs_matcher_set_current(self._h, ptrs, _ip(pitch),
                                               None if d is None else d.ctypes.data_as(C.POINTER(C.c_float)),
                                               0 if d is None else d.shape[1]))

    def set_current_disparity(self, disp):
        d = np.ascontiguousarray(disp, np.float32)
        self._ck(lib().svs_matcher_set_current(self._h, None, None, d.ctypes.data_as(C.POINTER(C.c_float)), d.shape[1]))

    def set_current_disparity_device(self, ptr, pitch):
        """cur_frame.disp from device memory, e.g. StereoMatcher.device_disparity()."""
        self._ck(lib().svs_matcher_set_disparity_device(self._h, ptr, pitch))

    def set_pyramid_device(self, which, ptrs, pitches, T_me_from_w=None):
        """which = -1: current frame, >= 0: keyframe slot (needs T_me_from_w); device pointers per level."""
        arr = (C.c_void_p * len(ptrs))(*ptrs)
        pitch = np.asarray(pitches, np.int32)
        T = None if T_me_from_w is None else np.ascontiguousarray(T_me_from_w, np.float64)
        self._ck(lib().svs_matcher_set_pyramid_device(self._h, which, None if T is None else _dp(T), arr, _ip(pitch)))

    def set_features(self, level, xy, content):
        xy = np.ascontiguousarray(xy, np.int32).reshape(-1, 2)
        content = np.ascontiguousarray(content, np.int32)
        self._ck(lib().svs_matcher_set_features(self._h, level, _ip(xy), _ip(content), len(xy)))

    def set_features_from_fast(self, level, fast_grid):
        """FAST corners of `fast_grid`'s last detect call, taken where they lie on the device."""
        self._ck(lib().svs_matcher_set_features_from_fast(self._h, level, fast_grid._h))

    def match(self, T_cur_from_actkey, T_actkey_from_w, points, search_radius, thr_mean, thr_std):
        """points: structured array with MATCH_POINT_DTYPE.  Returns a MATCH_RESULT_DTYPE array."""
        pts = np.ascontiguousarray(points, MATCH_POINT_DTYPE)
        out = np.zeros(len(pts), MATCH_RESULT_DTYPE)
        Ta = np.ascontiguousarray(T_cur_from_actkey, np.float64)
        Tb = np.ascontiguousarray(T_actkey_from_w, np.float64)
        rc = lib().svs_match(self._h, _dp(Ta), _dp(Tb), pts.ctypes.data_as(C.POINTER(SvsMatchPoint)), len(pts),
                             int(search_radius), int(thr_mean), int(thr_std),
                             out.ctypes.data_as(C.POINTER(SvsMatchResult)))
        if rc < 0:
            self._ck(rc)
        return out

    def match_track(self, T_cur_from_actkey, T_actkey_from_w, groups, num_max_points, search_radius, thr_mean, thr_std):
        """matchAndTrack's matching: groups = [newpoint_map[actkey], neighbours' newpoint_map lists ..., point_list],
        each a MATCH_POINT_DTYPE array.  Returns (MATCH_RESULT_DTYPE over all candidates, num_new_feat_matched,
        num_obs); entries of a neighbour group past the budget have matched = 0."""
        if len(groups) < 2:
            raise ValueError("groups: at least the active keyframe's new points and the neighbourhood's points")
        pts = np.ascontiguousarray(np.concatenate([np.asarray(g, MATCH_POINT_DTYPE) for g in groups]), MATCH_POINT_DTYPE)
        ends = np.cumsum([len(g) for g in groups]).astype(np.int32)
        out = np.zeros(len(pts), MATCH_RESULT_DTYPE)
        a, b = C.c_int(), C.c_int()
        self._ck(lib().svs_match_track(self._h, _dp(np.ascontiguousarray(T_cur_from_actkey, np.float64)),
                                       _dp(np.ascontiguousarray(T_actkey_from_w, np.float64)),
                                       pts.ctypes.data_as(C.POINTER(SvsMatchPoint)), len(pts), len(groups), _ip(ends),
                                       int(num_max_points), int(search_radius), int(thr_mean), int(thr_std),
                                       out.ctypes.data_as(C.POINTER(SvsMatchResult)), C.byref(a), C.byref(b)))
        return out, a.value, b.value

    def process_matched_points(self, T_cur_from_actkey, cam, n_new, params=None):
        """processMatchedPoints on the last match: returns (TRACKED_POINT_DTYPE gated entries, stats dict,
        add_flags [3, 3], drop_keyframe)."""
        p = params or frontend_params()
        out = np.zeros(self.max_points, TRACKED_POINT_DTYPE)   # room for every candidate of the last match
        st = SvsPointStats()
        flags = np.zeros(9, np.int32)
        drop = C.c_int()
        rc = lib().svs_processMatchedPoints(self._h, _dp(np.ascontiguousarray(T_cur_from_actkey, np.float64)),
                                            C.byref(SvsCam(*[float(x) for x in cam])), int(n_new), C.byref(p),
                                            out.ctypes.data, C.byref(st), _ip(flags), C.byref(drop))
        if rc < 0:
            self._ck(rc)
        return out[:rc], st.as_dict(), flags.reshape(3, 3), bool(drop.value)

    def add_more_points(self, fresh, cam, keyframe_slot, T_newkey_from_cur=None, params=None):
        """addNewPoints (fresh = 1) / addMorePoints (fresh = 0, after process_matched_points) on the current frame:
        returns (NEW_POINT_DTYPE points, MATCH_POINT_DTYPE rows, counts per level), in seeding order."""
        p = params or frontend_params()
        T = np.array([0, 0, 0, 1, 0, 0, 0], np.float64) if T_newkey_from_cur is None else \
            np.ascontiguousarray(T_newkey_from_cur, np.float64)
        cap = sum((p.num_max_points >> l) + 1 for l in range(self.nlevels))
        pts = np.zeros(cap, NEW_POINT_DTYPE)
        rows = np.zeros(cap, MATCH_POINT_DTYPE)
        counts = np.zeros(4, np.int32)
        rc = lib().svs_addMorePoints(self._h, int(fresh), _dp(T), C.byref(SvsCam(*[float(x) for x in cam])),
                                     int(keyframe_slot), C.byref(p), pts.ctypes.data, rows.ctypes.data, cap, _ip(counts))
        if rc < 0:
            self._ck(rc)
        return pts[:rc], rows[:rc], counts[:self.nlevels]


def shall_we_drop_new_keyframe(stats, T_cur_from_actkey, params=None):
    """svs_shallWeDropNewKeyframe on a stats dict of process_matched_points."""
    st = SvsPointStats()
    st.num_matched_points[:] = list(stats["num_matched_points"])
    st.grid2x2[:] = [int(x) for x in np.asarray(stats["grid2x2"]).reshape(-1)]
    st.grid3x3[:] = [int(x) for x in np.asarray(stats["grid3x3"]).reshape(-1)]
    st.av_track_length = float(stats["av_track_length"])
    st.num_tracked, st.num_new = int(stats["num_tracked"]), int(stats["num_new"])
    p = params or frontend_params()
    return bool(lib().svs_shallWeDropNewKeyframe(C.byref(st), _dp(np.ascontiguousarray(T_cur_from_actkey, np.float64)),
                                                 C.byref(p)))


class FramePreprocessor(_Handle):
    """FrameGrabber::preprocessing (reference frame_grabber.cpp:287-336) on the device: uint8 and
    float pyramids and the x/y derivatives of one frame; outputs stay on the GPU."""

    _destroy, _last_error = "svs_prep_destroy", "svs_prep_last_error"

    def __init__(self, w, h, nlevels=3, device=-1):
        self._open("svs_prep_create", device, w, h, nlevels)
        self.nlevels = nlevels

    def process(self, img):
        img = np.ascontiguousarray(img, np.uint8)
        self._ck(lib().svs_prep_process(self._h, img.ctypes.data_as(c_up), img.strides[0]))

    def level(self, l):
        """dict(w, h, u8, pitch_u8, f32, dx, dy, stride_f32) with raw device pointers."""
        w, h, p8, s32 = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        u8, f32, dx, dy = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        self._ck(lib().svs_prep_level(self._h, l, C.byref(w), C.byref(h), C.byref(u8), C.byref(p8), C.byref(f32),
                                      C.byref(dx), C.byref(dy), C.byref(s32)))
        return dict(w=w.value, h=h.value, u8=u8.value, pitch_u8=p8.value, f32=f32.value, dx=dx.value, dy=dy.value,
                    stride_f32=s32.value)

    def get_u8(self, l):
        lv = self.level(l)
        out = np.zeros((lv["h"], lv["w"]), np.uint8)
        self._ck(lib().svs_prep_get_u8(self._h, l, out.ctypes.data_as(c_up)))
        return out

    def get_f32(self, l, which=0):
        lv = self.level(l)
        out = np.zeros((lv["h"], lv["w"]), np.float32)
        self._ck(lib().svs_prep_get_f32(self._h, l, which, out.ctypes.data_as(C.POINTER(C.c_float))))
        return out


class StereoMatcher(_Handle):
    """StereoFrontend::calcDisparityCpu (reference stereo_frontend.cpp:620-653): cv::StereoBM with the reference's
    settings on the device, bit for bit OpenCV 4.x's output (svs_stereo_* in svs_b200.h).  The map stays on the GPU
    for the tracker and the matcher; disparity() reads it back."""

    _destroy, _last_error = "svs_stereo_destroy", "svs_stereo_last_error"

    def __init__(self, w, h, num_disparities=32, device=-1):
        self._open("svs_stereo_create", device, w, h, num_disparities)
        self.w, self.h, self.num_disparities = w, h, num_disparities

    def _image(self, img):
        """(pointer, pitch, on_device, keep-alive) of an (h, w) uint8 image: a numpy array (host), a
        FramePreprocessor.level() dict or a CUDA torch tensor (device)."""
        if isinstance(img, dict):
            if (img["w"], img["h"]) != (self.w, self.h):
                raise SvsError(-1, f"a {img['w']}x{img['h']} level for a {self.w}x{self.h} stereo handle")
            return img["u8"], img["pitch_u8"], 1, None
        if _is_torch_tensor(img) and img.is_cuda:
            import torch
            if img.dtype != torch.uint8 or tuple(img.shape) != (self.h, self.w) or img.stride(1) != 1:
                raise SvsError(-1, f"a device image must be a ({self.h}, {self.w}) torch.uint8 tensor with unit column "
                                   f"stride, not {img.dtype} {tuple(img.shape)}")
            torch.cuda.current_stream(img.device).synchronize()   # the handle reads the image on its own stream
            return img.data_ptr(), img.stride(0), 1, img
        a = np.ascontiguousarray(img)
        if a.dtype != np.uint8 or a.shape != (self.h, self.w):
            raise SvsError(-1, f"a host image must be a ({self.h}, {self.w}) uint8 array, not {a.dtype} {a.shape}")
        return a.ctypes.data, a.strides[0], 0, a

    def compute(self, left, right):
        """left / right: (h, w) uint8 numpy arrays, or device images (FramePreprocessor.level(0), CUDA tensors)."""
        lp, lpitch, ldev, lkeep = self._image(left)
        rp, rpitch, rdev, rkeep = self._image(right)
        self._ck(lib().svs_stereo_compute(self._h, lp, lpitch, ldev, rp, rpitch, rdev))

    def device_disparity(self):
        """(device pointer, floats per row) of the last map."""
        p, s = C.c_void_p(), C.c_int()
        self._ck(lib().svs_stereo_disparity(self._h, C.byref(p), C.byref(s)))
        return p.value, s.value

    def disparity(self):
        out = np.empty((self.h, self.w), np.float32)
        self._ck(lib().svs_stereo_get(self._h, out.ctypes.data_as(C.POINTER(C.c_float))))
        return out


class PoseOptimizer(_Handle):
    """BA_SE3_XYZ_STEREO (reference pose_optimizer.h:495): motion-only LM, whole loop in one kernel."""

    _destroy, _last_error = "svs_pose_destroy", "svs_pose_last_error"

    def __init__(self, max_obs=16384, device=-1):
        self._open("svs_pose_create", device, max_obs)

    @staticmethod
    def _params(robust_kernel, kernel_param, num_iter, initial_mu):
        return SvsPoseParams(int(robust_kernel), float(kernel_param), int(num_iter), float(initial_mu), 0.00001)

    @staticmethod
    def _stats(st):
        return dict(initial_chi2=st.initial_chi2, chi2=st.chi2, max_err=st.max_err, num_obs=st.num_obs,
                    iterations=st.iterations, trials=st.trials, ms=st.ms)

    def calc_fast_motion_only(self, obs_point_id, obs_uvu, point_xyz, cam, T_frame, robust_kernel=True,
                              kernel_param=1.0, num_iter=50, initial_mu=-1.0):
        """Returns (T_frame_new, stats); cam = (f, px, py, baseline).  obs_point_id, obs_uvu and point_xyz are numpy
        arrays, or CUDA torch tensors on the handle's device (then svs_calcFastMotionOnly_device reads them where they
        are; the current torch stream is synchronised first).  T_frame and the returned pose are host arrays [7]."""
        T = np.array(T_frame, np.float64).copy()
        c = SvsCam(*[float(x) for x in cam])
        p = self._params(robust_kernel, kernel_param, num_iter, initial_mu)
        st = SvsPoseStats()
        if any(_is_torch_tensor(a) for a in (obs_point_id, obs_uvu, point_xyz)):
            import torch
            arrs = []
            for name, a, dt in (("obs_point_id", obs_point_id, torch.int32), ("obs_uvu", obs_uvu, torch.float64),
                                ("point_xyz", point_xyz, torch.float64)):
                if not (isinstance(a, torch.Tensor) and a.is_cuda):
                    raise TypeError(f"{name}: a CUDA tensor (all three arrays of a device track are)")
                arrs.append(a.detach().to(dt).contiguous())
            pid, obs, xyz = arrs[0].reshape(-1), arrs[1].reshape(-1, 3), arrs[2].reshape(-1, 3)
            if not (pid.device == obs.device == xyz.device):
                raise ValueError("obs_point_id, obs_uvu and point_xyz: tensors on one device")
            torch.cuda.current_stream(pid.device).synchronize()   # the handle reads the arrays on its own stream
            self._ck(lib().svs_calcFastMotionOnly_device(self._h, pid.numel(), pid.data_ptr(), obs.data_ptr(), len(xyz),
                                                         xyz.data_ptr(), C.byref(c), C.byref(p), _dp(T), C.byref(st)))
        else:
            pid = np.ascontiguousarray(obs_point_id, np.int32)
            obs = np.ascontiguousarray(obs_uvu, np.float64).reshape(-1, 3)
            xyz = np.ascontiguousarray(point_xyz, np.float64).reshape(-1, 3)
            self._ck(lib().svs_calcFastMotionOnly(self._h, len(pid), _ip(pid), _dp(obs), len(xyz), _dp(xyz), C.byref(c),
                                                  C.byref(p), _dp(T), C.byref(st)))
        self.n, self.npoints = len(pid), len(xyz)
        return T, self._stats(st)

    # outputs of grad: name -> (trailing shape)
    _GRAD_OUT = {"obs": (3,), "xyz": (3,), "cam": ()}

    def grad(self, dL_dT, lam=0.0, want=("obs", "xyz", "cam")):
        """svs_pose_grad: dL/d(observations, points, camera) of the pose the last calc_fast_motion_only returned, from
        dL_dT [6] in the tangent (upsilon, omega) of T <- exp(delta) T (None = 0).  `want` names the outputs to compute,
        any of "obs" [n,3], "xyz" [npoints,3], "cam" [4] (f, px, py, b); the others are neither computed nor written.
        Returns (dict name -> array for the names in `want`, rc, stats); rc = 1: H + lam I is not positive definite
        (outputs zeroed).  Numpy in, numpy out; a CUDA float64 tensor on the handle's device in, tensors out (the current
        torch stream is synchronised first)."""
        bad = [w for w in want if w not in self._GRAD_OUT]
        if bad:
            raise ValueError(f"want: unknown outputs {bad} (choose from {list(self._GRAD_OUT)})")
        n, npts = getattr(self, "n", 0), getattr(self, "npoints", 0)
        shape = {"obs": (n, 3), "xyz": (npts, 3), "cam": (4,)}
        st = SvsPoseGradStats()
        if _is_torch_tensor(dL_dT):
            import torch
            if not (dL_dT.is_cuda and dL_dT.dtype == torch.float64):
                raise TypeError("dL_dT: a CUDA float64 tensor (or numpy, or None)")
            g = dL_dT.detach().reshape(6).contiguous()
            res = {w: torch.empty(shape[w], dtype=torch.float64, device=g.device) for w in want}
            torch.cuda.current_stream(g.device).synchronize()   # the handle reads the arrays on its own stream
            ptr = lambda t: t.data_ptr() if t is not None and t.numel() else None
            on_device = 1
        else:
            g = None if dL_dT is None else np.ascontiguousarray(np.asarray(dL_dT, np.float64).reshape(6))
            res = {w: np.zeros(shape[w]) for w in want}
            ptr = lambda a: a.ctypes.data if a is not None and a.size else None
            on_device = 0
        rc = lib().svs_pose_grad(self._h, float(lam), ptr(g), ptr(res.get("obs")), ptr(res.get("xyz")),
                                 ptr(res.get("cam")), on_device, C.byref(st))
        if rc < 0:
            self._ck(rc)
        return res, rc, st.as_dict()

    def calc_fast_motion_only_matched(self, matcher, cam, T_frame, robust_kernel=True, kernel_param=1.0, num_iter=50,
                                      initial_mu=-1.0):
        T = np.array(T_frame, np.float64).copy()
        c = SvsCam(*[float(x) for x in cam])
        p = self._params(robust_kernel, kernel_param, num_iter, initial_mu)
        st = SvsPoseStats()
        self._ck(lib().svs_calcFastMotionOnly_matched(self._h, matcher._h, C.byref(c), C.byref(p), _dp(T), C.byref(st)))
        return T, self._stats(st)


class DenseTrackerCpuVariant(_Handle):
    """DenseTracker as the reference builds it without SCAVISLAM_CUDA_SUPPORT (dense_tracking.cpp:222-423):
    denseTrackingCpu / computeDensePointCloudCpu semantics, executed on the GPU."""

    _destroy, _last_error = "svs_dtc_destroy", "svs_dtc_last_error"

    def __init__(self, w, h, nlevels=3, device=-1):
        self._open("svs_dtc_create", device, w, h, nlevels, why="no CUDA device, or a level size is not a multiple of 4")
        self.w, self.h, self.nlevels = w, h, nlevels

    @staticmethod
    def _cams(cams):
        arr = (SvsCam * len(cams))()
        for i, c in enumerate(cams):
            arr[i] = SvsCam(*[float(x) for x in c[:4]])
        return arr

    def set_prev_u8(self, level, img):
        img = np.ascontiguousarray(img, np.uint8)
        self._ck(lib().svs_dtc_set_prev_u8(self._h, level, img.ctypes.data, img.strides[0], 0))

    def set_prev_u8_device(self, level, ptr, pitch):
        self._ck(lib().svs_dtc_set_prev_u8(self._h, level, ptr, pitch, 1))

    def set_cur(self, level, cur, dx, dy):
        ims = [np.ascontiguousarray(x, np.float32) for x in (cur, dx, dy)]
        self._ck(lib().svs_dtc_set_cur(self._h, level, ims[0].ctypes.data, ims[1].ctypes.data, ims[2].ctypes.data,
                                       ims[0].shape[1], 0))

    def set_cur_device(self, level, cur, dx, dy, stride):
        self._ck(lib().svs_dtc_set_cur(self._h, level, cur, dx, dy, stride, 1))

    def set_disparity(self, disp):
        d = np.ascontiguousarray(disp, np.float32)
        self._ck(lib().svs_dtc_set_disparity(self._h, d.ctypes.data_as(C.POINTER(C.c_float)), d.shape[1]))

    def set_disparity_device(self, ptr, stride):
        """frame_data_->disp from device memory, e.g. StereoMatcher.device_disparity()."""
        self._ck(lib().svs_dtc_set_disparity_device(self._h, ptr, stride))

    def compute_point_cloud(self, T, cams):
        T = np.ascontiguousarray(T, np.float64)
        self._ck(lib().svs_computeDensePointCloudCpu(self._h, _dp(T), self._cams(cams)))

    def point_cloud(self, level):
        out = np.zeros(((self.h >> level) // 4, (self.w >> level) // 4, 4), np.float32)
        self._ck(lib().svs_dtc_get_point_cloud(self._h, level, out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def set_point_cloud(self, level, cloud):
        c = np.ascontiguousarray(cloud, np.float32)
        self._ck(lib().svs_dtc_set_point_cloud(self._h, level, c.ctypes.data_as(C.POINTER(C.c_float))))

    def track(self, T, cams):
        T = np.array(T, np.float64).copy()
        st = SvsDtStats()
        self._ck(lib().svs_denseTrackingCpu(self._h, self._cams(cams), _dp(T), C.byref(st)))
        return T, dict(chi2=list(st.chi2[:self.nlevels]), passes=list(st.passes[:self.nlevels]), ms_total=st.ms_total)


class ConstraintBuilder(_Handle):
    """SlamGraph::computeConstraint (reference slam_graph.cpp:785-846) for a batch of pose pairs."""

    _destroy, _last_error = "svs_constraints_destroy", "svs_constraints_last_error"

    def __init__(self, device=-1):
        self._open("svs_constraints_create", device)

    def compute(self, poses, feat_ptr, feat_point, point_anchor, xyz_anchor, v1, v2):
        """Returns (T_1_from_2[n,7], Lambda[n,6,6], visibility_strength[n])."""
        poses = np.ascontiguousarray(poses, np.float64).reshape(-1, 7)
        fp, fpt = np.ascontiguousarray(feat_ptr, np.int32), np.ascontiguousarray(feat_point, np.int32)
        pa = np.ascontiguousarray(point_anchor, np.int32)
        xyz = np.ascontiguousarray(xyz_anchor, np.float64).reshape(-1, 3)
        v1, v2 = np.ascontiguousarray(v1, np.int32), np.ascontiguousarray(v2, np.int32)
        n = len(v1)
        T, Lam, ns = np.zeros((n, 7)), np.zeros((n, 36)), np.zeros(n, np.int32)
        rc = lib().svs_computeConstraint_batch(self._h, len(poses), _dp(poses), _ip(fp), _ip(fpt), len(pa), _ip(pa), _dp(xyz),
                                               n, _ip(v1), _ip(v2), _dp(T), _dp(Lam), _ip(ns))
        self._ck(rc)
        return T, Lam.reshape(n, 6, 6), ns


class DeviceMap(_Handle):
    """The part of SlamGraph the optimiser reads, kept on the device (reference slam_graph.hpp:65-137), and
    copyDataToG2o (slam_graph.cpp:985-1032) as kernels feeding a BundleAdjuster."""

    _destroy, _last_error = "svs_map_destroy", "svs_map_last_error"

    def __init__(self, device=-1):
        self._open("svs_map_create", device)

    def set(self, poses, point_anchor, xyz_anchor, vis_ptr, vis_pose, feat_center, feat_level):
        poses = np.ascontiguousarray(poses, np.float64).reshape(-1, 7)
        pa = np.ascontiguousarray(point_anchor, np.int32)
        xyz = np.ascontiguousarray(xyz_anchor, np.float64).reshape(-1, 3)
        vp_, vs = np.ascontiguousarray(vis_ptr, np.int32), np.ascontiguousarray(vis_pose, np.int32)
        cen = np.ascontiguousarray(feat_center, np.float64).reshape(-1, 3)
        lvl = np.ascontiguousarray(feat_level, np.int32)
        self._ck(lib().svs_map_set(self._h, len(poses), _dp(poses), len(pa), _ip(pa), _dp(xyz), _ip(vp_), _ip(vs), _dp(cen),
                                   _ip(lvl)))
        self.V, self.Np = len(poses), len(pa)

    def update_poses(self, vertex, poses):
        v = np.ascontiguousarray(vertex, np.int32)
        T = np.ascontiguousarray(poses, np.float64).reshape(-1, 7)
        self._ck(lib().svs_map_update_poses(self._h, len(v), _ip(v), _dp(T)))

    def update_points(self, point, xyz_anchor):
        v = np.ascontiguousarray(point, np.int32)
        x = np.ascontiguousarray(xyz_anchor, np.float64).reshape(-1, 3)
        self._ck(lib().svs_map_update_points(self._h, len(v), _ip(v), _dp(x)))

    def get(self):
        """(poses [V,7], xyz_anchor [Np,3]) as they lie on the device."""
        T, x = np.zeros((self.V, 7)), np.zeros((max(self.Np, 1), 3))
        self._ck(lib().svs_map_get(self._h, _dp(T), _dp(x)))
        return T, x[:self.Np]

    def absorb(self, ba):
        """SlamGraph::restoreDataFromG2o, device to device: the optimised window of `ba` goes back into the map."""
        self._ck(lib().svs_map_absorb(self._h, ba._h))

    def set_graph(self, nbr_ptr, nbr_id, nbr_T=None, nbr_Lambda=None):
        """The pose graph: per vertex its neighbours, strongest first; optionally the marginalised constraint of every
        directed entry (T_nbr_from_me [7], Lambda [36])."""
        ptr, ids = np.ascontiguousarray(nbr_ptr, np.int32), np.ascontiguousarray(nbr_id, np.int32)
        T = None if nbr_T is None else np.ascontiguousarray(nbr_T, np.float64).reshape(-1, 7)
        Lm = None if nbr_Lambda is None else np.ascontiguousarray(nbr_Lambda, np.float64).reshape(-1, 36)
        self._nn = len(ids)
        self._ck(lib().svs_map_set_graph(self._h, _ip(ptr), _ip(ids), None if T is None else _dp(T), None if Lm is None else _dp(Lm)))

    def select_window(self, root, inner_window_size, double_window_size):
        """computeInitialDoubleWin + computeActivePointsAndExtendOuterWindow + the pair selection of copyContraintsToG2o
        on the device.  Returns dict(window_vertex, inner, active_point, c_i, c_j, c_T, c_Lambda)."""
        capP, capL, capC = self.V, max(self.Np, 1), max(getattr(self, "_nn", 0), 1)
        win, inner, act = np.zeros(capP, np.int32), np.zeros(capP, np.uint8), np.zeros(capL, np.int32)
        ci, cj, cT, cL = np.zeros(capC, np.int32), np.zeros(capC, np.int32), np.zeros((capC, 7)), np.zeros((capC, 36))
        P, L, Cn = C.c_int(), C.c_int(), C.c_int()
        self._ck(lib().svs_map_select_window(self._h, int(root), int(inner_window_size), int(double_window_size), capP, C.byref(P),
                                             _ip(win), inner.ctypes.data_as(c_up), capL, C.byref(L), _ip(act), capC, C.byref(Cn),
                                             _ip(ci), _ip(cj), _dp(cT), _dp(cL)))
        P, L, Cn = P.value, L.value, Cn.value
        return dict(window_vertex=win[:P].copy(), inner=inner[:P].copy(), active_point=act[:L].copy(), c_i=ci[:Cn].copy(),
                    c_j=cj[:Cn].copy(), c_T=cT[:Cn].copy(), c_Lambda=cL[:Cn].copy())

    @staticmethod
    def _keyframe_args(T_newkey_from_oldkey, new_anchor, new_xyz, new_anchor_center, new_anchor_level, new_center, new_level,
                       track_point, track_center, track_level):
        T = np.ascontiguousarray(T_newkey_from_oldkey, np.float64).reshape(7)
        na = np.ascontiguousarray(new_anchor, np.int32)
        d3 = lambda a, n: np.zeros((n, 3)) if a is None else np.ascontiguousarray(a, np.float64).reshape(n, 3)
        nx, nac, nc = d3(new_xyz, len(na)), d3(new_anchor_center, len(na)), d3(new_center, len(na))
        nal, nl = np.ascontiguousarray(new_anchor_level, np.int32), np.ascontiguousarray(new_level, np.int32)
        tp = np.ascontiguousarray(track_point, np.int32)
        tc, tl = d3(track_center, len(tp)), np.ascontiguousarray(track_level, np.int32)
        keep = (T, na, nx, nac, nal, nc, nl, tp, tc, tl)
        return keep, [_dp(T), len(na), _ip(na), _dp(nx), _dp(nac), _ip(nal), _dp(nc), _ip(nl), len(tp), _ip(tp), _dp(tc), _ip(tl)]

    def add_keyframe(self, oldkey, T_newkey_from_oldkey, new_anchor=(), new_xyz=None, new_anchor_center=None,
                     new_anchor_level=(), new_center=None, new_level=(), track_point=(), track_center=None, track_level=()):
        """SlamGraph::addKeyframe on the device tables.  Returns (index of the new vertex, index of the first new point)."""
        keep, args = self._keyframe_args(T_newkey_from_oldkey, new_anchor, new_xyz, new_anchor_center, new_anchor_level,
                                         new_center, new_level, track_point, track_center, track_level)
        v, q = C.c_int(), C.c_int()
        self._ck(lib().svs_map_add_keyframe(self._h, int(oldkey), *args, C.byref(v), C.byref(q)))
        self.V += 1
        self.Np += len(keep[1])
        return v.value, q.value

    def set_pose_graph(self, nbr_ptr, nbr_id, nbr_strength, nbr_T, nbr_Lambda):
        """The pose graph with the strength of every directed entry (each list strongest first) and its constraint
        (T_nbr_from_me [7], Lambda [36]): the graph add_keyframe_graph and add_edges grow."""
        ptr = np.ascontiguousarray(nbr_ptr, np.int32)
        ids, st = np.ascontiguousarray(nbr_id, np.int32), np.ascontiguousarray(nbr_strength, np.int32)
        T = np.ascontiguousarray(nbr_T, np.float64).reshape(-1, 7)
        Lm = np.ascontiguousarray(nbr_Lambda, np.float64).reshape(-1, 36)
        if not len(ids) == len(st) == len(T) == len(Lm):
            raise ValueError("nbr_id, nbr_strength, nbr_T and nbr_Lambda must have one row per entry")
        self._ck(lib().svs_map_set_pose_graph(self._h, _ip(ptr), _ip(ids), _ip(st), _dp(T), _dp(Lm)))
        self._nn = len(ids)

    def get_graph(self):
        """The pose graph as it lies on the device: dict(nbr_ptr, nbr_id, nbr_strength, nbr_T, nbr_Lambda)."""
        nn = C.c_int()
        self._ck(lib().svs_map_get_graph(self._h, 0, C.byref(nn), None, None, None, None, None))
        n = nn.value
        ptr, ids, st = np.zeros(self.V + 1, np.int32), np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32)
        T, Lm = np.zeros((max(n, 1), 7)), np.zeros((max(n, 1), 36))
        self._ck(lib().svs_map_get_graph(self._h, n, C.byref(nn), _ip(ptr), _ip(ids), _ip(st), _dp(T), _dp(Lm)))
        return dict(nbr_ptr=ptr, nbr_id=ids[:n], nbr_strength=st[:n], nbr_T=T[:n], nbr_Lambda=Lm[:n])

    def add_keyframe_graph(self, oldkey, T_newkey_from_oldkey, covis_thr, width, height, new_anchor=(), new_xyz=None,
                           new_anchor_center=None, new_anchor_level=(), new_center=None, new_level=(), track_point=(),
                           track_center=None, track_level=()):
        """The whole of SlamGraph::addKeyframe on the device: computeStrength (quirk B15 kept), the growth of add_keyframe
        and addNewEdges(LOCAL) with the constraints.  Returns (index of the new vertex, index of the first new point,
        strength table [n, 2] of (vertex, strength) rows in ascending vertex order, number of edges added)."""
        keep, args = self._keyframe_args(T_newkey_from_oldkey, new_anchor, new_xyz, new_anchor_center, new_anchor_level,
                                         new_center, new_level, track_point, track_center, track_level)
        v, q, nt, ne = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        table = np.zeros((max(self.V, 1), 2), np.int32)
        self._ck(lib().svs_map_add_keyframe_graph(self._h, int(oldkey), *args, int(covis_thr), int(width), int(height), C.byref(v),
                                                  C.byref(q), C.byref(nt), _ip(table), C.byref(ne)))
        self.V += 1
        self.Np += len(keep[1])
        self._nn = getattr(self, "_nn", 0) + 2 * ne.value
        return v.value, q.value, table[:nt.value].copy(), ne.value

    def add_edges(self, v1, v2, strength, moved_vertex=-1, T_moved_from_w=None):
        """registerKeyframes' / addLoopClosure's edges: (v1[k], v2[k]) with strength[k] into both lists, the constraint
        computeConstraint(v1, v2) with moved_vertex placed at T_moved_from_w."""
        a, b, s = (np.ascontiguousarray(x, np.int32) for x in (v1, v2, strength))
        if not len(a) == len(b) == len(s):
            raise ValueError("v1, v2 and strength must have one entry per edge")
        T = None if T_moved_from_w is None else np.ascontiguousarray(T_moved_from_w, np.float64).reshape(7)
        self._ck(lib().svs_map_add_edges(self._h, len(a), _ip(a), _ip(b), _ip(s), int(moved_vertex), None if T is None else _dp(T)))
        self._nn = getattr(self, "_nn", 0) + 2 * len(a)

    def prepare_for_optimization(self, root, loop, inner_window_size, double_window_size):
        """SlamGraph::prepareForOptimization(root, loop) on the device: the window of select_window, reinitializePoses,
        unmargPosesEnteringInnerW and margPosesLeftInnerWindow.  Returns select_window's dict, its constraints read after
        the marginalisation, plus do_optimization (P >= 2)."""
        capP, capL, capC = self.V, max(self.Np, 1), max(getattr(self, "_nn", 0), 1)
        win, inner, act = np.zeros(capP, np.int32), np.zeros(capP, np.uint8), np.zeros(capL, np.int32)
        ci, cj, cT, cL = np.zeros(capC, np.int32), np.zeros(capC, np.int32), np.zeros((capC, 7)), np.zeros((capC, 36))
        P, L, Cn, do = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        self._ck(lib().svs_map_prepare_for_optimization(self._h, int(root), int(loop), int(inner_window_size), int(double_window_size),
                                                        C.byref(do), capP, C.byref(P), _ip(win), inner.ctypes.data_as(c_up), capL,
                                                        C.byref(L), _ip(act), capC, C.byref(Cn), _ip(ci), _ip(cj), _dp(cT), _dp(cL)))
        P, L, Cn = P.value, L.value, Cn.value
        return dict(window_vertex=win[:P].copy(), inner=inner[:P].copy(), active_point=act[:L].copy(), c_i=ci[:Cn].copy(),
                    c_j=cj[:Cn].copy(), c_T=cT[:Cn].copy(), c_Lambda=cL[:Cn].copy(), do_optimization=bool(do.value))

    def window_state(self):
        """(window_type [V] uint8: 0 outside, 1 INNER, 2 OUTER -- the last prepare's window; marginalized [nnzN] uint8:
        Edge::is_marginalized of each directed entry in get_graph's order)."""
        nn = C.c_int()
        self._ck(lib().svs_map_get_window_state(self._h, 0, C.byref(nn), None, None))
        n = nn.value
        wt, mg = np.zeros(max(self.V, 1), np.uint8), np.zeros(max(n, 1), np.uint8)
        self._ck(lib().svs_map_get_window_state(self._h, n, C.byref(nn), wt.ctypes.data_as(c_up), mg.ctypes.data_as(c_up)))
        return wt[:self.V].copy(), mg[:n].copy()

    def set_problem(self, ba, window_vertex, active_point, cam, fixed=None, c_i=(), c_j=(), c_T=None, c_Lambda=None):
        """Assembles the window on the device and loads it into `ba` (a BundleAdjuster).  Returns E."""
        win = np.ascontiguousarray(window_vertex, np.int32)
        act = np.ascontiguousarray(active_point, np.int32)
        fx = None if fixed is None else np.ascontiguousarray(fixed, np.uint8)
        ci, cj = np.ascontiguousarray(c_i, np.int32), np.ascontiguousarray(c_j, np.int32)
        cT = np.zeros((0, 7)) if c_T is None else np.ascontiguousarray(c_T, np.float64)
        cL = np.zeros((0, 36)) if c_Lambda is None else np.ascontiguousarray(c_Lambda, np.float64)
        cm = SvsCam(*[float(x) for x in cam])
        E = C.c_int()
        self._ck(lib().svs_ba_set_problem_from_map(ba._h, self._h, len(win), _ip(win),
                                                   None if fx is None else fx.ctypes.data_as(c_up), len(act), _ip(act),
                                                   len(ci), _ip(ci), _ip(cj), _dp(cT), _dp(cL), C.byref(cm), C.byref(E)))
        ba.P, ba.L, ba.E, ba.C = len(win), len(act), E.value, len(ci)
        return E.value

    def last_edges(self, E):
        ep, es, ea = np.zeros(E, np.int32), np.zeros(E, np.int32), np.zeros(E, np.int32)
        obs, info = np.zeros((E, 3)), np.zeros((E, 3))
        self._ck(lib().svs_map_last_edges(self._h, E, _ip(ep), _ip(es), _ip(ea), _dp(obs), _dp(info)))
        return ep, es, ea, obs, info

    def global_loop_closure(self, matcher, pose, cam, covis_thr, query, loop, T_query_from_loop, window_vertex, vertex_slot,
                            cap=None):
        """Backend::globalLoopClosure on the device (svs_globalLoopClosure): `matcher` (a GuidedMatcher) holds the loop
        keyframe as its current frame and the keyframe pyramids in the slots vertex_slot names, `pose` is a
        PoseOptimizer.  Returns (result dict, tracks dict(point, uvu, level)); a verified loop has grown the map."""
        win = np.ascontiguousarray(window_vertex, np.int32)
        slot = np.ascontiguousarray(vertex_slot, np.int32)
        Tq = np.ascontiguousarray(T_query_from_loop, np.float64).reshape(7)
        cap = max(self.Np, 1) if cap is None else int(cap)
        tp, tu, tl = np.zeros(max(cap, 1), np.int32), np.zeros((max(cap, 1), 3)), np.zeros(max(cap, 1), np.int32)
        r = SvsLoopResult()
        cm = SvsCam(*[float(x) for x in cam])
        rc = lib().svs_globalLoopClosure(self._h, matcher._h, pose._h, C.byref(cm), int(covis_thr), int(query), int(loop),
                                         _dp(Tq), len(win), _ip(win), _ip(slot), C.byref(r), cap, _ip(tp), _dp(tu), _ip(tl))
        out = {f: getattr(r, f) for f in ("verified", "stage", "n_candidates", "n_matched1", "n_matched2", "n_tracks",
                                          "num_left", "num_right", "num_upper", "num_lower")}
        for f in ("T_align1", "T_newloop_from_oldloop", "T_newloop_from_w"):
            out[f] = np.array(getattr(r, f)[:])
        out["lm"] = [PoseOptimizer._stats(r.lm[k]) for k in range(2)]
        if rc != 0:
            err = self._error(rc)
            err.result = out
            raise err
        n = out["n_tracks"] if out["stage"] in (0, 3, 4) else 0
        return out, dict(point=tp[:n].copy(), uvu=tu[:n].copy(), level=tl[:n].copy())

    def local_register_frame(self, matcher, pose, cam, covis_thr, root, window_vertex, vertex_slot, cap_stats=None,
                             cap_tracks=None):
        """Backend::localRegisterFrame on the device (svs_localRegisterFrame): `matcher` (a GuidedMatcher) holds the root
        keyframe as its current frame and the keyframe pyramids in the slots vertex_slot names, `pose` is a
        PoseOptimizer; the pose graph must be set (set_graph).  Returns (result dict, stats [REGISTER_STATS_DTYPE] in
        ascending vertex order, tracks dict(point, uvu, level, committed) in match order); a registered frame has grown
        the map.  A refused call raises SvsError with the result dict as .result."""
        win = np.ascontiguousarray(window_vertex, np.int32)
        slot = np.ascontiguousarray(vertex_slot, np.int32)
        cs = max(self.V, 1) if cap_stats is None else int(cap_stats)
        ct = max(self.Np, 1) if cap_tracks is None else int(cap_tracks)
        st = np.zeros(max(cs, 1), REGISTER_STATS_DTYPE)
        tp, tu = np.zeros(max(ct, 1), np.int32), np.zeros((max(ct, 1), 3))
        tl, tc = np.zeros(max(ct, 1), np.int32), np.zeros(max(ct, 1), np.int32)
        r = SvsRegisterResult()
        cm = SvsCam(*[float(x) for x in cam])
        rc = lib().svs_localRegisterFrame(self._h, matcher._h, pose._h, C.byref(cm), int(covis_thr), int(root), len(win), _ip(win),
                                          _ip(slot), C.byref(r), cs, st.ctypes.data, ct, _ip(tp), _dp(tu), _ip(tl), _ip(tc))
        out = {f: getattr(r, f) for f in REGISTER_COUNTS}
        for f in ("T_align1", "T_newroot_from_oldroot", "T_newroot_from_w"):
            out[f] = np.array(getattr(r, f)[:])
        out["lm"] = [PoseOptimizer._stats(r.lm[k]) for k in range(2)]
        if rc != 0:
            err = self._error(rc)
            err.result = out
            raise err
        gated = out["stage"] in (0, 4)
        nt, ns = (out["n_tracks"], out["n_stats"]) if gated else (0, 0)
        return out, st[:ns].copy(), dict(point=tp[:nt].copy(), uvu=tu[:nt].copy(), level=tl[:nt].copy(), committed=tc[:nt].copy())


def load_surf_vocabulary(path):
    """The reference's vocabulary file (surfwords10000.png: every float stored as four uint8 of an 8-bit image,
    placerecognizer.cpp:91-100) as float32 [W][64]."""
    import cv2
    img = cv2.imread(str(path), -1)
    if img is None or img.dtype != np.uint8 or img.ndim != 2 or img.shape[1] % 4:
        raise ValueError(f"{path}: not a single-channel 8-bit image with a multiple of 4 columns")
    return np.ascontiguousarray(img).view(np.float32).copy()


class PlaceRecognizer(_Handle):
    """PlaceRecognizer::addLocation (reference placerecognizer.cpp:206-324) on the device: words, TF-IDF loop
    candidates, brute-force match and the RANSAC check.  Semantics: include/svs_b200.h (svs_place)."""

    _destroy, _last_error = "svs_place_destroy", "svs_place_last_error"

    def __init__(self, words, cam, device=-1):
        words = np.ascontiguousarray(words, np.float32).reshape(-1, 64)
        self._open("svs_place_create", device, len(words), words.ctypes.data_as(C.POINTER(C.c_float)),
                   C.byref(SvsCam(*[float(x) for x in cam])))
        self._last_n = 0

    def _ck(self, rc):
        """Counts are results here: only a negative value is an error."""
        if rc < 0:
            raise self._error(rc)
        return rc

    @property
    def num_places(self):
        return self._ck(lib().svs_place_num_places(self._h))

    def add_location(self, keyframe_id, desc, uvu, do_loop_detection=True, exclude=(), num_ransac=100, pixel_thr=2.5,
                     seed=0):
        """Returns dict(best_keyframe_id, best_score, num_matches, num_inliers, loop_found, T_query_from_loop[7], ms,
        inlier_query, inlier_train)."""
        desc = np.ascontiguousarray(desc, np.float32).reshape(-1, 64)
        uvu = np.ascontiguousarray(uvu, np.float64).reshape(-1, 3)
        if len(uvu) != len(desc):
            raise ValueError("desc and uvu need one row per descriptor")
        n = len(desc)
        ex = np.ascontiguousarray(list(exclude), np.int32)
        p = SvsPlaceParams(int(num_ransac), float(pixel_thr), int(seed) & (2 ** 64 - 1))
        r = SvsPlaceResult()
        iq, it = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32)
        self._ck(lib().svs_place_add_location(self._h, int(keyframe_id), n, desc.ctypes.data_as(C.POINTER(C.c_float)),
                                              _dp(uvu), int(bool(do_loop_detection)), len(ex), _ip(ex), C.byref(p),
                                              C.byref(r), _ip(iq), _ip(it)))
        self._last_n = n
        ni = r.num_inliers
        return dict(best_keyframe_id=r.best_keyframe_id, best_score=r.best_score, num_matches=r.num_matches,
                    num_inliers=ni, loop_found=bool(r.loop_found), T_query_from_loop=np.array(r.T_query_from_loop[:]),
                    ms=r.ms, inlier_query=iq[:ni].copy(), inlier_train=it[:ni].copy())

    def last_words(self):
        w = np.zeros(max(self._last_n, 1), np.int32)
        n = self._ck(lib().svs_place_last_words(self._h, _ip(w)))
        return w[:n].copy()

    def last_scores(self):
        cap = max(self.num_places, 1)
        ids, sc = np.zeros(cap, np.int32), np.zeros(cap, np.float32)
        n = self._ck(lib().svs_place_last_scores(self._h, cap, _ip(ids), sc.ctypes.data_as(C.POINTER(C.c_float))))
        return ids[:n].copy(), sc[:n].copy()

    def last_matches(self):
        t, d = np.zeros(max(self._last_n, 1), np.int32), np.zeros(max(self._last_n, 1), np.float32)
        n = self._ck(lib().svs_place_last_matches(self._h, _ip(t), d.ctypes.data_as(C.POINTER(C.c_float))))
        return t[:n].copy(), d[:n].copy()

    def last_hypotheses(self):
        """(triple[H, 3], inliers[H], best): -1 marks a void hypothesis; best = -1 when none had an inlier."""
        b = C.c_int()
        H = self._ck(lib().svs_place_last_hypotheses(self._h, 0, None, None, C.byref(b)))
        tri, inl = np.zeros((max(H, 1), 3), np.int32), np.zeros(max(H, 1), np.int32)
        self._ck(lib().svs_place_last_hypotheses(self._h, H, _ip(tri), _ip(inl), C.byref(b)))
        return tri[:H].copy(), inl[:H].copy(), b.value
