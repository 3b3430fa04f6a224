"""ctypes bindings of liblsdreg.so (include/lsdreg.h) and thin numpy / torch front-ends.

The product path is the CUDA library: importing this module fails loudly when liblsdreg.so has not
been built, and every call raises :class:`LsdError` when no CUDA device is present.  There is no
CPU fallback and nothing here imports ``oracle/``.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblsdreg.so")

OK, NO_EFFECTIVE_POINTS, SCAN_TOO_SMALL, MAP_SEEDED = 0, 1, 2, 3
MAP_SATURATED = 6
ERR_INVALID, ERR_CUDA, ERR_NO_DEVICE, ERR_CAPACITY, ERR_GRID_OVERFLOW, ERR_IO = -1, -2, -3, -4, -5, -6
STENCIL_CENTER, STENCIL_NEARBY6, STENCIL_NEARBY18, STENCIL_NEARBY26, STENCIL_NEARBY74, STENCIL_EXACT = 0, 6, 18, 26, 74, 1000


class LsdError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"lsdreg status {status}: {msg}")
        self.status = status


class LioParams(C.Structure):
    _fields_ = [("max_points", C.c_int), ("max_scan_points", C.c_int), ("filter_size_surf", C.c_float),
                ("filter_size_map", C.c_float), ("ivox_resolution", C.c_float), ("ivox_nearby", C.c_int),
                ("map_log2_lines", C.c_int), ("max_iterations", C.c_int), ("laser_point_cov", C.c_double),
                ("converge_eps", C.c_double), ("degenerate_detect_en", C.c_int), ("knn_mode_exact", C.c_int), ("eskf_literal", C.c_int), ("async_map_insert", C.c_int)]


class LioInfo(C.Structure):
    _fields_ = [("n_down", C.c_int), ("iterations", C.c_int), ("n_eff", C.c_int), ("degenerate", C.c_int),
                ("n_added", C.c_int), ("converged", C.c_int), ("res_mean", C.c_double), ("gpu_ms", C.c_double),
                ("kernel_launches", C.c_int)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class RegParams(C.Structure):
    _fields_ = [("kind", C.c_int), ("resolution", C.c_double), ("ndt_neighbors", C.c_int), ("max_iterations", C.c_int),
                ("transformation_epsilon", C.c_double), ("rotation_epsilon_deg", C.c_double), ("lm_max_iterations", C.c_int),
                ("lm_init_lambda_factor", C.c_double), ("max_process_time_us", C.c_int64), ("k_correspondences", C.c_int),
                ("max_corr_dist", C.c_double), ("normal_search_sq", C.c_double), ("map_resolution", C.c_double),
                ("map_log2_lines", C.c_int)]


REG_NDT_P2D, REG_GICP, REG_VGICP = 0, 1, 2


class LoopParams(C.Structure):
    _fields_ = [("distance_thresh", C.c_double), ("accum_distance_thresh", C.c_double),
                ("distance_from_last_edge_thresh", C.c_double), ("distance_new_keyframe_thresh", C.c_double),
                ("distance_keyframe_thresh", C.c_double), ("fitness_score_max_range", C.c_double),
                ("fitness_score_thresh", C.c_double), ("coarse", RegParams), ("accurate", RegParams)]


class LoopResult(C.Structure):
    _fields_ = [("key1", C.c_int32), ("key2", C.c_int32), ("relpose16", C.c_float * 16), ("coarse_score", C.c_double),
                ("score", C.c_double), ("information36", C.c_double * 36), ("n_candidates", C.c_int32)]


class LoopReport(C.Structure):
    _fields_ = [("new_slot", C.c_int32), ("decision", C.c_int32), ("n_candidates", C.c_int32), ("best_slot", C.c_int32),
                ("best_score", C.c_double)]


class GalignParams(C.Structure):
    _fields_ = [("reg", RegParams), ("sc_dist_thres", C.c_double), ("icp_score_thres", C.c_double),
                ("fitness_score_max_range", C.c_double), ("max_batch_points", C.c_int64), ("sc_db_capacity", C.c_int)]


class GalignClosure(C.Structure):
    _fields_ = [("ref_slot", C.c_int32), ("new_slot", C.c_int32), ("relpose16", C.c_float * 16), ("score", C.c_double),
                ("sc_dist", C.c_float), ("sc_yaw", C.c_float)]


class GalignMatch(C.Structure):
    _fields_ = [("new_slot", C.c_int32), ("ref_slot", C.c_int32), ("sc_dist", C.c_float), ("sc_yaw", C.c_float),
                ("converged", C.c_int32), ("iterations", C.c_int32), ("score", C.c_double), ("accepted", C.c_int32)]


class OverlapParams(C.Structure):
    _fields_ = [("distance_thresh", C.c_double), ("candidate_link_dist", C.c_int32), ("max_candidate_num", C.c_int32),
                ("fitness_score_max_range", C.c_double), ("fitness_score_thresh", C.c_double),
                ("fitness_inlier_thresh", C.c_double), ("inlier_max_range", C.c_double), ("filter_range", C.c_double),
                ("filter_min_z", C.c_float), ("coarse", RegParams), ("accurate", RegParams)]


class OverlapResult(C.Structure):
    _fields_ = [("key1", C.c_int32), ("key2", C.c_int32), ("relpose16", C.c_double * 16), ("score", C.c_double),
                ("coarse_score", C.c_double)]


class OverlapReport(C.Structure):
    _fields_ = [("new_slot", C.c_int32), ("decision", C.c_int32), ("n_candidates", C.c_int32), ("n_prescreened", C.c_int32),
                ("best_slot", C.c_int32), ("n_accum", C.c_int32), ("accum_incomplete", C.c_int32), ("best_score", C.c_double),
                ("score", C.c_double)]


# what OverlapDetector.detect decided for each new key frame (LSD_OVERLAP_*)
OVERLAP_NO_CANDIDATES, OVERLAP_NO_MATCH, OVERLAP_GICP_DIVERGED, OVERLAP_GICP_REJECT, OVERLAP_FOUND = range(5)


# what LoopDetector.detect decided for each new key frame (LSD_LOOP_*)
LOOP_SKIPPED, LOOP_NO_CANDIDATES, LOOP_COARSE_REJECT, LOOP_GICP_DIVERGED, LOOP_GICP_REJECT, LOOP_FOUND = range(6)


class ImuParams(C.Structure):
    _fields_ = [("ext_R", C.c_double * 9), ("ext_t", C.c_double * 3), ("gyr_cov", C.c_double), ("acc_cov", C.c_double),
                ("b_gyr_cov", C.c_double), ("b_acc_cov", C.c_double), ("undistort", C.c_int)]


class VfeParams(C.Structure):
    _fields_ = [("min_range", C.c_float * 3), ("max_range", C.c_float * 3), ("voxel_size", C.c_float * 3),
                ("max_points_per_voxel", C.c_int), ("max_voxels", C.c_int), ("max_points", C.c_int), ("num_feature", C.c_int),
                ("max_frame_num", C.c_int), ("unordered_ids", C.c_int)]

class FloorParams(C.Structure):
    _fields_ = [("prefilter_leaf", C.c_float), ("distance_near", C.c_double), ("distance_far", C.c_double),
                ("clip_keep_d", C.c_float), ("clip_cut_d", C.c_float), ("use_normal_filtering", C.c_int), ("normal_k", C.c_int),
                ("normal_filter_deg", C.c_double), ("viewpoint_z", C.c_float), ("ransac_threshold", C.c_double),
                ("ransac_probability", C.c_double), ("ransac_max_iterations", C.c_int), ("floor_pts_thresh", C.c_int),
                ("floor_normal_deg", C.c_double), ("hypotheses_per_batch", C.c_int)]


class FloorResult(C.Structure):
    _fields_ = [("found", C.c_int32), ("reason", C.c_int32), ("coeffs", C.c_float * 4), ("n_input", C.c_int32),
                ("n_prefiltered", C.c_int32), ("n_clipped", C.c_int32), ("n_candidates", C.c_int32), ("n_inliers", C.c_int32),
                ("map_dropped", C.c_int32), ("iterations", C.c_int32), ("skipped", C.c_int32), ("best_hypothesis", C.c_int32),
                ("batches", C.c_int32), ("hypotheses_scored", C.c_int64), ("launches", C.c_int32), ("round_trips", C.c_int32)]


# lsd_floor_default_params presets, FloorResult.reason and the stages of FloorDetector.cloud (LSD_FLOOR_*)
FLOOR_MAPPING, FLOOR_GROUND, FLOOR_RENDER = range(3)
FLOOR_FOUND, FLOOR_EMPTY, FLOOR_FEW_CANDIDATES, FLOOR_NO_MODEL, FLOOR_FEW_INLIERS, FLOOR_NOT_VERTICAL = range(6)
FLOOR_STAGES = {"prefiltered": 0, "clipped": 1, "candidates": 2, "inliers": 3}

# every symbol include/lsdreg.h declares: (name, restype, argtypes)
_vp, _i, _f, _d = C.c_void_p, C.c_int, C.c_float, C.c_double
_pp = C.POINTER(C.c_void_p)
_pi = C.POINTER(C.c_int)
_pu64 = C.POINTER(C.c_uint64)
SIGNATURES = [
    ("lsd_version", C.c_char_p, []),
    ("lsd_last_error", C.c_char_p, []),
    ("lsd_init", _i, [_i]),
    ("lsd_map_create", _i, [_pp, _f, _i]),
    ("lsd_map_destroy", _i, [_vp]),
    ("lsd_map_clear", _i, [_vp]),
    ("lsd_map_set_shard", _i, [_vp, _i, _i, _i, _i]),
    ("lsd_map_insert", _i, [_vp, _vp, _i, C.c_int32]),
    ("lsd_map_insert_dev", _i, [_vp, _vp, _i, C.c_int32]),
    ("lsd_map_stats", _i, [_vp, _pu64, _pu64, _pu64]),
    ("lsd_map_delete_boxes", _i, [_vp, _vp, _i, _pu64]),
    ("lsd_map_stream", _i, [_vp, C.POINTER(C.c_void_p)]),
    ("lsd_knn_query", _i, [_vp, _vp, _i, _i, _f, _i, _vp, _vp, _vp]),
    ("lsd_knn_query_dev", _i, [_vp, _vp, _i, _i, _f, _i, _vp, _vp, _vp]),
    ("lsd_knn_set_shape", _i, [_vp, _i]),
    ("lsd_map_enable_lru", _i, [_vp, C.c_uint64, _d]),
    ("lsd_map_set_travel_distance", _i, [_vp, _d]),
    ("lsd_map_dump", _i, [_vp, _vp, _vp, _vp, _vp, C.c_uint64, _pu64]),
    ("lsd_map_evict", _i, [_vp, _vp]),
    ("lsd_map_saturated", _i, [_vp, _pi, _vp]),
    ("lsd_map_enable_bricks", _i, [_vp, _i]),
    ("lsd_map_brick_stats", _i, [_vp, _vp, _vp, _vp]),
    ("lsd_voxelgrid_create", _i, [_pp, _i, _i]),
    ("lsd_voxelgrid_destroy", _i, [_vp]),
    ("lsd_voxelgrid_filter", _i, [_vp, _vp, _i, _f, _vp, _pi]),
    ("lsd_voxelgrid_filter_dev", _i, [_vp, _vp, _i, _f, _vp, _vp]),
    ("lsd_lio_default_params", None, [C.POINTER(LioParams)]),
    ("lsd_lio_create", _i, [_pp, C.POINTER(LioParams)]),
    ("lsd_lio_destroy", _i, [_vp]),
    ("lsd_lio_map", _vp, [_vp]),
    ("lsd_lio_set_nearby", _i, [_vp, _i]),
    ("lsd_lio_set_ekf_inited", _i, [_vp, _i]),
    ("lsd_lio_set_stale_rows", _i, [_vp, _i]),
    ("lsd_lio_set_reference_order", _i, [_vp, _i]),
    ("lsd_lio_reference_order_fallbacks", _i, [_vp, _vp]),
    ("lsd_debug_nth_element", _i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    ("lsd_debug_esti_plane", _i, [_vp, _i, _f, _vp, _vp]),
    ("lsd_lio_set_knn_shape", _i, [_vp, _i]),
    ("lsd_lio_set_pdl", _i, [_vp, _i]),
    ("lsd_lio_shard_exchange_stats", _i, [_vp, C.POINTER(_d), C.POINTER(C.c_longlong)]),
    ("lsd_lio_set_pipeline", _i, [_vp, _i]),
    ("lsd_lio_pipeline_stats", _i, [_vp, _vp, _vp]),
    ("lsd_lio_prefetch_dev", _i, [_vp, _vp, _i]),
    ("lsd_lio_set_next_id", _i, [_vp, C.c_int32]),
    ("lsd_lio_shard_export", _i, [_vp, _i, _i, _i, _i, _vp]),
    ("lsd_lio_shard_connect", _i, [_vp, _vp]),
    ("lsd_lio_sync", _i, [_vp, C.POINTER(_d), _pi]),
    ("lsd_lio_set_profile", _i, [_vp, _i]),
    ("lsd_lio_get_profile", _i, [_vp, _vp, _vp]),
    ("lsd_lio_load_scan", _i, [_vp, _vp, _i, _i, _pi]),
    ("lsd_lio_load_scan_dev", _i, [_vp, _vp, _i, _i, _pi]),
    ("lsd_lio_get_down", _i, [_vp, _vp, _i, _pi]),
    ("lsd_lio_linearize", _i, [_vp, _vp, _i, _vp, _vp, C.POINTER(_d), _pi, _pi]),
    ("lsd_lio_get_matches", _i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    ("lsd_lio_update", _i, [_vp, _vp, _vp, C.POINTER(LioInfo)]),
    ("lsd_lio_map_incremental", _i, [_vp, _vp, _pi]),
    ("lsd_lio_get_map_flags", _i, [_vp, _vp, _i, _pi, C.POINTER(_d)]),
    ("lsd_lio_scan", _i, [_vp, _vp, _i, _vp, _vp, C.POINTER(LioInfo)]),
    ("lsd_lio_scan_dev", _i, [_vp, _vp, _i, _vp, _vp, C.POINTER(LioInfo)]),
    ("lsd_lio_prefetch", _i, [_vp, _vp, _i]),
    ("lsd_reg_default_params", None, [C.POINTER(RegParams), _i]),
    ("lsd_reg_create", _i, [_pp, C.POINTER(RegParams)]),
    ("lsd_reg_destroy", _i, [_vp]),
    ("lsd_reg_set_target", _i, [_vp, _vp, _i]),
    ("lsd_reg_set_target_dev", _i, [_vp, _vp, _i]),
    ("lsd_reg_set_source", _i, [_vp, _vp, _i]),
    ("lsd_reg_set_source_dev", _i, [_vp, _vp, _i]),
    ("lsd_reg_set_max_correspondence_distance", _i, [_vp, _d]),
    ("lsd_reg_align", _i, [_vp, _vp, _vp, _pi, _pi]),
    ("lsd_reg_get_final", _i, [_vp, _vp, _vp]),
    ("lsd_reg_fitness", _i, [_vp, _vp, _d, C.POINTER(_d)]),
    ("lsd_reg_cost", _i, [_vp, _vp, _i, _vp, _vp, C.POINTER(_d), _pi]),
    ("lsd_reg_get_correspondences", _i, [_vp, _vp, _i, _pi]),
    ("lsd_reg_stats", _i, [_vp, _pi, C.POINTER(C.c_longlong)]),
    ("lsd_reg_get_covariances", _i, [_vp, _i, _vp]),
    ("lsd_reg_get_voxels", _i, [_vp, _i, _vp, _vp, _vp, _vp, _pi]),
    ("lsd_reg_iteration_log", _i, [_vp, _vp, _i, _pi]),
    ("lsd_reg_shard_export", _i, [_vp, _i, _i, _i, _vp]),
    ("lsd_reg_shard_connect", _i, [_vp, _vp]),
    ("lsd_loop_default_params", None, [C.POINTER(LoopParams)]),
    ("lsd_loop_create", _i, [_pp, C.POINTER(LoopParams)]),
    ("lsd_loop_destroy", _i, [_vp]),
    ("lsd_loop_add_keyframe", _i, [_vp, _vp, _i, _d, C.POINTER(C.c_int32)]),
    ("lsd_loop_detect", _i, [_vp, _vp, _vp, _i, _vp, _i, _vp, _i, _pi]),
    ("lsd_loop_last_reports", _i, [_vp, _vp, _i, _pi]),
    ("lsd_loop_last_edge", _i, [_vp, C.POINTER(_d), _i]),
    ("lsd_loop_find_candidates", _i, [C.POINTER(LoopParams), _d, _vp, _vp, _vp, _i, C.c_int32, _vp, _vp, _i, _pi]),
    ("lsd_loop_match", _i, [_vp, C.c_int32, _vp, _vp, _i, _vp, _vp, _vp, _vp, C.POINTER(C.c_longlong), _pi]),
    ("lsd_loop_iteration_log", _i, [_vp, _i, _vp, _i, _pi]),
    ("lsd_loop_fitness", _i, [_vp, C.c_int32, C.c_int32, _vp, _d, C.POINTER(_d), _pi]),
    ("lsd_loop_information_matrix", None, [_d, _vp]),
    ("lsd_galign_default_params", None, [C.POINTER(GalignParams)]),
    ("lsd_galign_create", _i, [_pp, C.POINTER(GalignParams)]),
    ("lsd_galign_destroy", _i, [_vp]),
    ("lsd_galign_add_keyframe", _i, [_vp, _vp, _i, _i, C.POINTER(C.c_int32)]),
    ("lsd_galign_search", _i, [_vp, _vp, _i, _vp, _i, _pi]),
    ("lsd_galign_last_matches", _i, [_vp, _vp, _i, _pi]),
    ("lsd_galign_last_stats", _i, [_vp, C.POINTER(C.c_longlong), _pi, _pi]),
    ("lsd_galign_set_max_batch_points", _i, [_vp, C.c_int64]),
    ("lsd_galign_merge_candidates", _i, [_vp, _vp, _vp, _vp, _i, _d, _vp, _vp, _vp, _i, _pi]),
    ("lsd_galign_match", _i, [_vp, C.c_int32, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, C.POINTER(C.c_longlong), _pi]),
    ("lsd_galign_iteration_log", _i, [_vp, _i, _vp, _i, _pi]),
    ("lsd_galign_cost", _i, [_vp, C.c_int32, C.c_int32, _vp, _i, _vp, _vp, C.POINTER(_d), _pi]),
    ("lsd_overlap_default_params", None, [C.POINTER(OverlapParams)]),
    ("lsd_overlap_create", _i, [_pp, C.POINTER(OverlapParams)]),
    ("lsd_overlap_destroy", _i, [_vp]),
    ("lsd_overlap_add_keyframe", _i, [_vp, _vp, _i, C.c_int32, C.POINTER(C.c_int32)]),
    ("lsd_overlap_detect", _i, [_vp, _vp, _vp, _i, _vp, _i, _vp, _i, _vp, _i, _pi]),
    ("lsd_overlap_last_reports", _i, [_vp, _vp, _i, _pi]),
    ("lsd_overlap_last_stats", _i, [_vp, C.POINTER(C.c_longlong), _pi, _pi, _pi]),
    ("lsd_overlap_release_targets", _i, [_vp]),
    ("lsd_overlap_find_candidates", _i, [C.POINTER(OverlapParams), _vp, _vp, _i, _vp, _i, _vp, _i, C.c_int32, _vp, _i, _pi]),
    ("lsd_overlap_guess", None, [_vp, _vp, _vp]),
    ("lsd_overlap_finetune_guess", None, [_vp, _vp]),
    ("lsd_overlap_fitness", _i, [_vp, C.c_int32, C.c_int32, _vp, _d, C.POINTER(_d), C.POINTER(_d), _pi, _pi, _pi]),
    ("lsd_overlap_match", _i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, C.POINTER(C.c_longlong), _pi]),
    ("lsd_overlap_iteration_log", _i, [_vp, _i, _vp, _i, _pi]),
    ("lsd_vfe_default_params", None, [C.POINTER(VfeParams)]),
    ("lsd_vfe_create", _i, [_pp, C.POINTER(VfeParams)]),
    ("lsd_vfe_destroy", _i, [_vp]),
    ("lsd_vfe_accumulate", _i, [_vp, _vp, _i, _vp, _i, _pi]),
    ("lsd_vfe_voxelize", _i, [_vp, _i, _pi]),
    ("lsd_vfe_get_output", _i, [_vp, _vp, _vp, _vp]),
    ("lsd_vfe_get_output_dev", _i, [_vp, _pp, _pp, _pp]),
    ("lsd_vfe_get_points", _i, [_vp, _vp, _i, _pi]),
    ("lsd_imu_default_params", None, [C.POINTER(ImuParams)]),
    ("lsd_imu_create", _i, [_pp, C.POINTER(ImuParams)]),
    ("lsd_imu_destroy", _i, [_vp]),
    ("lsd_imu_reset", _i, [_vp]),
    ("lsd_imu_is_init", _i, [_vp, _pi]),
    ("lsd_imu_process", _i, [_vp, _vp, _i, _vp, _d, _d, _vp, _vp, _i, _vp, _vp, _pi]),
    ("lsd_imu_process_dev", _i, [_vp, _vp, _i, _vp, _d, _d, _vp, _vp, _i, _vp, _vp, _pi]),
    ("lsd_imu_get_cloud_dev", _i, [_vp, _pp, _pi, _pp]),
    ("lsd_imu_get_cloud", _i, [_vp, _vp, _i, _pi]),
    ("lsd_imu_get_poses", _i, [_vp, _vp, _i, _pi]),
    ("lsd_eskf_predict", _i, [_vp, _vp, _d, _vp, _vp, _vp]),
    ("lsd_imu_get_start_state", _i, [_vp, _vp, C.POINTER(_d)]),
    ("lsd_fastlio_create", _i, [_pp, _vp, _vp, _i, _i, _d, _i]),
    ("lsd_fastlio_set_capacity", _i, [_vp, _i, _i]),
    ("lsd_fastlio_destroy", _i, [_vp]),
    ("lsd_fastlio_imu_enqueue", _i, [_vp, _d, _vp, _vp]),
    ("lsd_fastlio_ins_enqueue", _i, [_vp, _i, _i, C.c_uint64, _vp, _d, _d, _d]),
    ("lsd_fastlio_pcl_enqueue", _i, [_vp, _vp, _vp, _i, C.c_uint64]),
    ("lsd_fastlio_main", _i, [_vp]),
    ("lsd_fastlio_odometry", _i, [_vp, _vp, _vp]),
    ("lsd_fastlio_state", _i, [_vp, _vp]),
    ("lsd_fastlio_is_init", _i, [_vp]),
    ("lsd_fastlio_last", _i, [_vp, _pi, C.POINTER(LioInfo)]),
    ("lsd_fastlio_get_filter", _i, [_vp, _vp, _vp]),
    ("lsd_fastlio_lio", _vp, [_vp]),
    ("lsd_fastlio_pop_package", _i, [_vp, C.POINTER(_d), C.POINTER(_d), _pi, _vp, _vp, _i, _pi, _vp, _i, _pi, _vp]),
    ("lsd_sc_create", _i, [_pp, _i]),
    ("lsd_sc_destroy", _i, [_vp]),
    ("lsd_sc_make", _i, [_vp, _vp, _i, _vp, _i, _vp, _vp, _vp]),
    ("lsd_sc_make_dev", _i, [_vp, _vp, _i, _vp, _i, _vp, _vp, _vp]),
    ("lsd_sc_db_clear", _i, [_vp]),
    ("lsd_sc_db_add", _i, [_vp, _vp, _i]),
    ("lsd_sc_db_add_made", _i, [_vp, _i]),
    ("lsd_sc_db_size", _i, [_vp, _pi]),
    ("lsd_sc_query", _i, [_vp, _vp, _i, _vp, _vp, _vp, _vp]),
    ("lsd_sc_distance", _i, [_vp, _vp, _vp, _i, _vp, _vp]),
    ("lsd_sc_detect_closest", _i, [_vp, _i, _d, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(_d)]),
    ("lsd_sc_detect_candidates", _i, [_vp, _i, _d, _vp, _vp, _vp, C.POINTER(C.c_int32)]),
    ("lsd_localmap_create", _i, [_pp, _d, _d]),
    ("lsd_localmap_destroy", _i, [_vp]),
    ("lsd_localmap_add_keyframe", _i, [_vp, _vp, _i, _vp]),
    ("lsd_localmap_update", _i, [_vp, _vp, _pi, _pi, C.POINTER(_d)]),
    ("lsd_localmap_get_dev", _i, [_vp, _pp, _pi]),
    ("lsd_localmap_get", _i, [_vp, _vp, _i, _pi]),
    ("lsd_keyframe_filter", _i, [_vp, _i, _f, _i, _f, _f, _vp, _pi]),
    ("lsd_keyframe_filter_dev", _i, [_vp, _i, _f, _i, _f, _f, _vp, _pi]),
    ("lsd_keyframe_save", _i, [C.c_char_p, C.c_uint64, C.c_int64, _vp, _i, _vp]),
    ("lsd_keyframe_load", _i, [C.c_char_p, _pu64, C.POINTER(C.c_int64), _vp, _vp, _i, _pi]),
    ("lsd_floor_default_params", None, [C.POINTER(FloorParams), _i]),
    ("lsd_floor_create", _i, [_pp, C.POINTER(FloorParams)]),
    ("lsd_floor_destroy", _i, [_vp]),
    ("lsd_floor_detect", _i, [_vp, _vp, _i, C.POINTER(FloorResult)]),
    ("lsd_floor_detect_dev", _i, [_vp, _vp, _i, C.POINTER(FloorResult)]),
    ("lsd_floor_get_cloud", _i, [_vp, _i, _vp, _i, _pi]),
    ("lsd_floor_get_cloud_dev", _i, [_vp, _i, _pp, _pi]),
    ("lsd_floor_get_normals", _i, [_vp, _vp, _vp, _i, _pi]),
    ("lsd_floor_last_samples", _i, [_vp, _vp, _vp, _vp, _i, _pi]),
    ("lsd_ransac_replay", _i, [_vp, _vp, _i, _i, _d, _i, _pi, _pi, _pi, _pi]),
    ("lsd_lio_init_cov", None, [_vp]),
    ("lsd_state_boxplus", None, [_vp, _vp]),
    ("lsd_state_boxminus", None, [_vp, _vp, _vp]),
    ("lsd_eskf_update_table", _i, [_vp, _vp, _vp, _vp, _vp, _i, _d, _i, _d, _i, _vp]),
]


def load_library(path: str = LIB_PATH) -> C.CDLL:
    if not os.path.exists(path):
        raise ImportError(f"{path} not found: build it with `python __graft_entry__.py` "
                          "(nvcc, sm_90a). lsdreg has no CPU fallback.")
    lib = C.CDLL(path)
    for name, res, args in SIGNATURES:
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    return lib


lib = load_library()


def check(status: int) -> int:
    if status < 0:
        raise LsdError(status, lib.lsd_last_error().decode())
    return status


def _ptr(a) -> int:
    """Address of a numpy array's data or of a torch tensor's storage (host or device)."""
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return a.data_ptr()


def _f32(a) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.ndim != 2 or a.shape[1] != 4:
        raise ValueError("points must be float32 [n,4] = (x, y, z, intensity)")
    return a


def init(device: int = 0):
    check(lib.lsd_init(device))


class HashVoxelMap:
    """Device-resident hash-voxel map: the replacement of faster_lio::IVox (ivox3d.h)."""

    def __init__(self, resolution: float = 0.5, log2_lines: int = 20, _borrow: int | None = None):
        self._own = _borrow is None
        if _borrow is not None:
            self.h = C.c_void_p(_borrow)
        else:
            self.h = C.c_void_p()
            check(lib.lsd_map_create(C.byref(self.h), resolution, log2_lines))

    def close(self):
        if self._own and self.h:
            lib.lsd_map_destroy(self.h)
        self.h = None

    __del__ = close

    def clear(self):
        check(lib.lsd_map_clear(self.h))

    def insert(self, pts, id0: int = 0):
        """IVox::AddPoints.  numpy [n,4] (host path) or a CUDA torch tensor [n,4] (device path)."""
        if isinstance(pts, np.ndarray):
            pts = _f32(pts)
            check(lib.lsd_map_insert(self.h, _ptr(pts), pts.shape[0], id0))
        else:
            check(lib.lsd_map_insert_dev(self.h, _ptr(pts), pts.shape[0], id0))

    def stats(self):
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        check(lib.lsd_map_stats(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return dict(cells=a.value, points=b.value, dropped=c.value)

    def delete_boxes(self, boxes) -> int:
        """KD_TREE::Delete_Point_Boxes: boxes [n,6] = (min xyz, max xyz); returns the number of points deleted."""
        b = np.ascontiguousarray(np.asarray(boxes, np.float32).reshape(-1, 6))
        n = C.c_uint64()
        check(lib.lsd_map_delete_boxes(self.h, _ptr(b), b.shape[0], C.byref(n)))
        return int(n.value)

    def stream(self) -> int:
        """cudaStream_t (as an integer) the map's device calls run on."""
        p = C.c_void_p()
        check(lib.lsd_map_stream(self.h, C.byref(p)))
        return p.value or 0

    def knn(self, q, k: int = 5, max_sq: float = 5.0, stencil: int = STENCIL_NEARBY18):
        """IVox::GetClosestPoint for a batch -> (idx [nq,k], d2 [nq,k], cnt [nq]), canonical order."""
        q = _f32(q)
        nq = q.shape[0]
        idx = np.empty((nq, k), np.int32)
        d2 = np.empty((nq, k), np.float32)
        cnt = np.empty(nq, np.int32)
        check(lib.lsd_knn_query(self.h, _ptr(q), nq, k, max_sq, stencil, _ptr(idx), _ptr(d2), _ptr(cnt)))
        return idx, d2, cnt

    KNN_AUTO, KNN_WARP, KNN_THREAD, KNN_FLAT = 0, 1, 2, 3

    def enable_lru(self, capacity: int = 100000, max_distance: float = 100.0):
        """iVox's capacity + LRU eviction (include/lsdreg.h::lsd_map_enable_lru; laserMapping.cpp:1063-1064 runs 100 000 / 100 m)."""
        check(lib.lsd_map_enable_lru(self.h, int(capacity), float(max_distance)))

    def set_travel_distance(self, d: float):
        check(lib.lsd_map_set_travel_distance(self.h, float(d)))

    def dump(self):
        """Every stored point (include/lsdreg.h::lsd_map_dump) -> dict of voxel [n,3] int32, xyz [n,3] float32, id [n]
        int32, tombstone [n] bool; voxel by voxel, each voxel's points in storage order.  Copies the whole table."""
        n = C.c_uint64()
        check(lib.lsd_map_dump(self.h, None, None, None, None, 0, C.byref(n)))
        m = max(n.value, 1)
        vox = np.empty((m, 3), np.int32)
        xyz = np.empty((m, 3), np.float32)
        ids = np.empty(m, np.int32)
        tomb = np.empty(m, np.uint8)
        check(lib.lsd_map_dump(self.h, _ptr(vox), _ptr(xyz), _ptr(ids), _ptr(tomb), n.value, C.byref(n)))
        k = n.value
        return dict(voxel=vox[:k], xyz=xyz[:k], id=ids[:k], tombstone=tomb[:k].astype(bool))

    def evict(self) -> int:
        n = C.c_uint64()
        check(lib.lsd_map_evict(self.h, C.byref(n)))
        return n.value

    def saturated(self):
        f, n = C.c_int(), C.c_uint64()
        check(lib.lsd_map_saturated(self.h, C.byref(f), C.byref(n)))
        return bool(f.value), n.value

    def enable_bricks(self, log2_bricks: int = 16):
        """Also keep every point brick by brick (include/lsdreg.h::lsd_map_enable_bricks): batched k-NN shape 3 (TMA-staged pages)."""
        check(lib.lsd_map_enable_bricks(self.h, int(log2_bricks)))

    def brick_stats(self):
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        check(lib.lsd_map_brick_stats(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return dict(pages=a.value, replicas=b.value, dropped=c.value)

    def set_knn_shape(self, shape: int):
        """How a batch is mapped onto the GPU (include/lsdreg.h::lsd_knn_set_shape); results do not depend on it."""
        check(lib.lsd_knn_set_shape(self.h, int(shape)))

    def knn_dev(self, q, idx, d2, cnt, k: int = 5, max_sq: float = 5.0, stencil: int = STENCIL_NEARBY18):
        """Device-pointer variant on CUDA torch tensors; asynchronous."""
        check(lib.lsd_knn_query_dev(self.h, _ptr(q), q.shape[0], k, max_sq, stencil, _ptr(idx), _ptr(d2), _ptr(cnt)))


class VoxelGrid:
    """pcl::VoxelGrid replacement (centroid per leaf, ascending leaf index)."""

    def __init__(self, max_points: int = 400000, log2_max_cells: int = 28):
        self.h = C.c_void_p()
        check(lib.lsd_voxelgrid_create(C.byref(self.h), max_points, log2_max_cells))

    def close(self):
        if self.h:
            lib.lsd_voxelgrid_destroy(self.h)
        self.h = None

    __del__ = close

    def filter(self, pts: np.ndarray, leaf: float = 0.5) -> np.ndarray:
        pts = _f32(pts)
        out = np.empty_like(pts)
        m = C.c_int()
        st = lib.lsd_voxelgrid_filter(self.h, _ptr(pts), pts.shape[0], leaf, _ptr(out), C.byref(m))
        if st == ERR_GRID_OVERFLOW:  # PCL: warns and returns the input cloud
            return out[:m.value].copy()
        check(st)
        return out[:m.value].copy()


STATE_DIM, DOF = 26, 23


def init_cov() -> np.ndarray:
    P = np.zeros((DOF, DOF))
    lib.lsd_lio_init_cov(_ptr(P))
    return P


def make_state(pos=(0, 0, 0), rot_xyzw=(0, 0, 0, 1), off_R_xyzw=(0, 0, 0, 1), off_T=(0, 0, 0), vel=(0, 0, 0),
               bg=(0, 0, 0), ba=(0, 0, 0), grav=(0, 0, -9.809)) -> np.ndarray:
    return np.concatenate([pos, rot_xyzw, off_R_xyzw, off_T, vel, bg, ba, grav]).astype(np.float64)


def debug_nth_element(dist: np.ndarray, first: int, nth: int, last: int):
    """std::nth_element as the search kernel replays it (include/lsdreg.h lsd_debug_nth_element) -> (perm, path)."""
    d = np.ascontiguousarray(dist, np.float32)
    perm = np.empty(d.shape[0], np.int32)
    path = C.c_int()
    check(lib.lsd_debug_nth_element(_ptr(d), d.shape[0], first, nth, last, _ptr(perm), C.byref(path)))
    return perm, path.value


def debug_esti_plane(pts5: np.ndarray, thr: float = 0.1):
    """The LIO search's plane fit on the device, one thread per 5-point set (include/lsdreg.h lsd_debug_esti_plane)
    -> (pabcd [n,4] float32, ok [n] int32)."""
    p = np.ascontiguousarray(pts5, np.float32).reshape(-1, 5, 3)
    n = p.shape[0]
    pabcd = np.empty((n, 4), np.float32)
    ok = np.empty(n, np.int32)
    check(lib.lsd_debug_esti_plane(_ptr(p), n, thr, _ptr(pabcd), _ptr(ok)))
    return pabcd, ok


def state_boxplus(x: np.ndarray, d: np.ndarray) -> np.ndarray:
    x = np.array(x, np.float64)
    d = np.ascontiguousarray(d, np.float64)
    lib.lsd_state_boxplus(_ptr(x), _ptr(d))
    return x


def state_boxminus(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(a, np.float64)
    b = np.ascontiguousarray(b, np.float64)
    r = np.zeros(DOF)
    lib.lsd_state_boxminus(_ptr(a), _ptr(b), _ptr(r))
    return r


class Voxelizer:
    """Detection voxelizer: Preprocess (multi-frame window) + Voxelization (mean VFE, fp16)."""

    def __init__(self, **kw):
        self.h = None
        self.params = VfeParams()
        lib.lsd_vfe_default_params(C.byref(self.params))
        for k, v in kw.items():
            if not hasattr(self.params, k):
                raise TypeError(f"unknown voxelizer parameter {k}")
            if k in ("min_range", "max_range", "voxel_size"):
                v = (C.c_float * 3)(*v)
            setattr(self.params, k, v)
        self.h = C.c_void_p()
        check(lib.lsd_vfe_create(C.byref(self.h), C.byref(self.params)))

    def close(self):
        if self.h:
            lib.lsd_vfe_destroy(self.h)
        self.h = None

    __del__ = close

    def accumulate(self, points: np.ndarray, motion=None, realtime: bool = True) -> int:
        points = np.ascontiguousarray(points, np.float32)
        assert points.ndim == 2 and points.shape[1] == self.params.num_feature
        m = np.ascontiguousarray(np.eye(4) if motion is None else motion, np.float32)
        tot = C.c_int()
        check(lib.lsd_vfe_accumulate(self.h, _ptr(points), points.shape[0], _ptr(m), int(realtime), C.byref(tot)))
        return tot.value

    def points(self) -> np.ndarray:
        tot = C.c_int()
        check(lib.lsd_vfe_get_points(self.h, None, 0, C.byref(tot)))
        out = np.empty((tot.value, self.params.num_feature), np.float32)
        check(lib.lsd_vfe_get_points(self.h, _ptr(out), tot.value, C.byref(tot)))
        return out

    def voxelize(self, order_zyx: bool = True):
        nv = C.c_int()
        check(lib.lsd_vfe_voxelize(self.h, int(order_zyx), C.byref(nv)))
        V = nv.value
        feat = np.empty((V, self.params.num_feature), np.float16)
        idx = np.empty((V, 4), np.uint32)
        npts = np.empty(V, np.uint32)
        check(lib.lsd_vfe_get_output(self.h, _ptr(feat), _ptr(idx), _ptr(npts)))
        return feat, idx, npts


class Matcher:
    """Scan matcher with the call protocol of pcl::Registration (what select_registration_method()
    returns in the reference): set_target / set_source / align / has_converged / final / fitness."""

    def __init__(self, kind: str = "NDT_CUDA", **kw):
        self.h = None
        kinds = {"NDT_CUDA": REG_NDT_P2D, "NDT": REG_NDT_P2D, "FAST_GICP": REG_GICP, "GICP": REG_GICP,
                 "FAST_VGICP": REG_VGICP, "FAST_VGICP_CUDA": REG_VGICP, "VGICP": REG_VGICP}
        if kind not in kinds:
            raise ValueError(f"unknown registration method {kind}")
        self.params = RegParams()
        lib.lsd_reg_default_params(C.byref(self.params), kinds[kind])
        for k, v in kw.items():
            if not hasattr(self.params, k):
                raise TypeError(f"unknown matcher parameter {k}")
            setattr(self.params, k, v)
        self.h = C.c_void_p()
        check(lib.lsd_reg_create(C.byref(self.h), C.byref(self.params)))
        self.converged, self.iterations = False, 0
        self._n_tgt = self._n_src = 0

    def close(self):
        if self.h:
            lib.lsd_reg_destroy(self.h)
        self.h = None

    __del__ = close

    def iteration_log(self) -> np.ndarray:
        """[n_iter, 4] = (|t|_inf of the step, its rotation in degrees, cost at the linearisation, lambda) of the last align()."""
        n = C.c_int()
        check(lib.lsd_reg_iteration_log(self.h, None, 0, C.byref(n)))
        out = np.zeros((max(n.value, 1), 4))
        check(lib.lsd_reg_iteration_log(self.h, _ptr(out), n.value, C.byref(n)))
        return out[:n.value]

    def shard_export(self, rank: int, world: int, tile_cells: int = 32) -> np.ndarray:
        """Tile-sharded NDT target (include/lsdreg.h "Tile-sharded matcher"): this rank's blob for the all-gather."""
        blob = np.zeros(192, np.uint8)   # LSD_SHARD_BLOB_BYTES
        check(lib.lsd_reg_shard_export(self.h, rank, world, tile_cells, _ptr(blob)))
        return blob

    def shard_connect(self, blobs: np.ndarray):
        blobs = np.ascontiguousarray(blobs, np.uint8)
        check(lib.lsd_reg_shard_connect(self.h, _ptr(blobs)))

    def set_target(self, pts):
        if isinstance(pts, np.ndarray):
            pts = _f32(pts)
            check(lib.lsd_reg_set_target(self.h, _ptr(pts), pts.shape[0]))
        else:
            check(lib.lsd_reg_set_target_dev(self.h, _ptr(pts), pts.shape[0]))
        self._n_tgt = pts.shape[0]

    def set_target_ptr(self, dev_ptr: int, n: int):
        """setInputTarget from a raw device pointer (e.g. LocalMap.cloud_dev())."""
        check(lib.lsd_reg_set_target_dev(self.h, C.c_void_p(dev_ptr), n))
        self._n_tgt = n

    def set_source(self, pts):
        if isinstance(pts, np.ndarray):
            pts = _f32(pts)
            check(lib.lsd_reg_set_source(self.h, _ptr(pts), pts.shape[0]))
        else:
            check(lib.lsd_reg_set_source_dev(self.h, _ptr(pts), pts.shape[0]))
        self._n_src = pts.shape[0]

    def set_max_correspondence_distance(self, d: float):
        check(lib.lsd_reg_set_max_correspondence_distance(self.h, d))

    def align(self, guess=None) -> np.ndarray:
        g = np.ascontiguousarray(np.eye(4) if guess is None else guess, np.float32)
        out = np.zeros((4, 4), np.float32)
        cv, it = C.c_int(), C.c_int()
        check(lib.lsd_reg_align(self.h, _ptr(g), _ptr(out), C.byref(cv), C.byref(it)))
        self.converged, self.iterations = bool(cv.value), it.value
        return out

    def final(self):
        T, H = np.zeros((4, 4)), np.zeros((6, 6))
        check(lib.lsd_reg_get_final(self.h, _ptr(T), _ptr(H)))
        return T, H

    def fitness(self, max_range: float = 25.0, T=None) -> float:
        sc = C.c_double()
        Tp = None if T is None else np.ascontiguousarray(T, np.float64)
        check(lib.lsd_reg_fitness(self.h, None if Tp is None else _ptr(Tp), max_range, C.byref(sc)))
        return sc.value

    def cost(self, T, update: bool = True, deriv: bool = True):
        T = np.ascontiguousarray(T, np.float64)
        H, b = np.zeros((6, 6)), np.zeros(6)
        e, nc = C.c_double(), C.c_int()
        check(lib.lsd_reg_cost(self.h, _ptr(T), int(update), _ptr(H) if deriv else None, _ptr(b) if deriv else None,
                               C.byref(e), C.byref(nc)))
        return e.value, H, b, nc.value

    def correspondences(self) -> np.ndarray:
        """Correspondences of the last linearisation (GICP: target indices; NDT / VGICP: voxel slots), -1 = none."""
        n = C.c_int()
        check(lib.lsd_reg_get_correspondences(self.h, None, 0, C.byref(n)))
        out = np.empty(n.value, np.int32)
        check(lib.lsd_reg_get_correspondences(self.h, _ptr(out), n.value, C.byref(n)))
        return out

    def stats(self):
        nv, ln = C.c_int(), C.c_longlong()
        check(lib.lsd_reg_stats(self.h, C.byref(nv), C.byref(ln)))
        return dict(n_voxels=nv.value, launches=ln.value)

    def covariances(self, target: bool = True) -> np.ndarray:
        """[n, 4] = (smallest-eigenvalue direction of the k-NN covariance, neighbour count) of the target or source cloud."""
        n = self._n_tgt if target else self._n_src
        out = np.zeros((n, 4))
        check(lib.lsd_reg_get_covariances(self.h, int(target), _ptr(out)))
        return out

    def voxels(self) -> dict:
        """Every occupied line of the target voxel table: coord [m, 3], count [m], mean [m, 3], second [m, 6] (VGICP: mean
        covariance xx xy xz yy yz zz; NDT: the smallest-eigenvalue direction in 0..2)."""
        n = C.c_int()
        check(lib.lsd_reg_get_voxels(self.h, 0, None, None, None, None, C.byref(n)))
        m = n.value
        coord, count = np.zeros((m, 3), np.int32), np.zeros(m, np.int32)
        mean, second = np.zeros((m, 3)), np.zeros((m, 6))
        check(lib.lsd_reg_get_voxels(self.h, m, _ptr(coord), _ptr(count), _ptr(mean), _ptr(second), C.byref(n)))
        return dict(coord=coord, count=count, mean=mean, second=second)


def _loop_params(**kw) -> LoopParams:
    p = LoopParams()
    lib.lsd_loop_default_params(C.byref(p))
    for k, v in kw.items():
        if k in ("coarse", "accurate"):          # dict of lsd_reg_params_t fields
            for kk, vv in v.items():
                if not hasattr(p.coarse, kk):
                    raise TypeError(f"unknown matcher parameter {kk}")
                setattr(getattr(p, k), kk, vv)
        elif hasattr(p, k):
            setattr(p, k, v)
        else:
            raise TypeError(f"unknown loop-detector parameter {k}")
    return p


def _slots(a) -> np.ndarray:
    return np.ascontiguousarray(a, np.int32).reshape(-1)


def _poses(a) -> np.ndarray:
    a = np.ascontiguousarray(a, np.float64)
    if a.ndim != 3 or a.shape[1:] != (4, 4):
        raise ValueError("poses must be float64 [n_slots, 4, 4]")
    return a


class LoopDetector:
    """hdl_graph_slam::LoopDetector (loop_detector.hpp) on the device: key frames are added once (their clouds stay in
    device memory, addressed by slot); detect() finds candidates, aligns all of them to the new key frame with batched
    NDT, refines the best with GICP and returns the loops with their information matrices."""

    def __init__(self, **kw):
        self.h = None
        self.params = _loop_params(**kw)
        self.h = C.c_void_p()
        check(lib.lsd_loop_create(C.byref(self.h), C.byref(self.params)))
        self.accum = []

    def close(self):
        if self.h:
            lib.lsd_loop_destroy(self.h)
        self.h = None

    __del__ = close

    def add_keyframe(self, pts, accum_distance: float) -> int:
        pts = _f32(pts)
        slot = C.c_int32()
        check(lib.lsd_loop_add_keyframe(self.h, _ptr(pts), pts.shape[0], float(accum_distance), C.byref(slot)))
        self.accum.append(float(accum_distance))
        return slot.value

    @property
    def last_edge_accum_distance(self) -> float:
        v = C.c_double()
        check(lib.lsd_loop_last_edge(self.h, C.byref(v), 1))
        return v.value

    @last_edge_accum_distance.setter
    def last_edge_accum_distance(self, value: float):
        v = C.c_double(value)
        check(lib.lsd_loop_last_edge(self.h, C.byref(v), 0))

    def detect(self, poses, keyframes, new_keyframes) -> list[dict]:
        """poses: graph estimate of every slot [n_slots, 4, 4]; keyframes / new_keyframes: slots.  One dict per loop."""
        P, kf, nk = _poses(poses), _slots(keyframes), _slots(new_keyframes)
        cap = max(len(nk), 1)
        out = (LoopResult * cap)()
        n = C.c_int()
        check(lib.lsd_loop_detect(self.h, _ptr(P), _ptr(kf), kf.size, _ptr(nk), nk.size, out, cap, C.byref(n)))
        return [dict(key1=r.key1, key2=r.key2, relpose=np.array(r.relpose16, np.float32).reshape(4, 4),
                     coarse_score=r.coarse_score, score=r.score, information=np.array(r.information36).reshape(6, 6),
                     n_candidates=r.n_candidates) for r in out[:n.value]]

    def reports(self) -> list[dict]:
        """What the last detect() decided for each new key frame (decision: LOOP_*)."""
        n = C.c_int()
        check(lib.lsd_loop_last_reports(self.h, None, 0, C.byref(n)))
        out = (LoopReport * max(n.value, 1))()
        check(lib.lsd_loop_last_reports(self.h, out, n.value, C.byref(n)))
        return [dict(new_slot=r.new_slot, decision=r.decision, n_candidates=r.n_candidates, best_slot=r.best_slot,
                     best_score=r.best_score) for r in out[:n.value]]

    def find_candidates(self, poses, keyframes, new_slot: int, last_edge_accum_distance: float | None = None, accum=None):
        """find_candidates + the initial guesses (pure host).  Returns (slots [c], guesses [c, 4, 4])."""
        return find_loop_candidates(poses, self.accum if accum is None else accum, keyframes, new_slot,
                                    self.last_edge_accum_distance if last_edge_accum_distance is None else last_edge_accum_distance,
                                    params=self.params)

    def match(self, target_slot: int, candidates, guesses) -> dict:
        """The coarse stage alone for an explicit candidate list (parity tap)."""
        cand = _slots(candidates)
        n = cand.size
        G = np.ascontiguousarray(guesses, np.float64).reshape(n, 4, 4)
        T = np.zeros((n, 4, 4)); cv = np.zeros(n, np.int32); it = np.zeros(n, np.int32); fit = np.zeros(n)
        ln, rd = C.c_longlong(), C.c_int()
        check(lib.lsd_loop_match(self.h, int(target_slot), _ptr(cand), _ptr(G), n, _ptr(T), _ptr(cv), _ptr(it), _ptr(fit),
                                 C.byref(ln), C.byref(rd)))
        logs = []
        for i in range(n):
            m = C.c_int()
            check(lib.lsd_loop_iteration_log(self.h, i, None, 0, C.byref(m)))
            lg = np.zeros((max(m.value, 1), 4))
            check(lib.lsd_loop_iteration_log(self.h, i, _ptr(lg), m.value, C.byref(m)))
            logs.append(lg[:m.value])
        return dict(final=T, converged=cv.astype(bool), iterations=it, fitness=fit, launches=ln.value, rounds=rd.value,
                    iteration_logs=logs)

    def fitness(self, target_slot: int, source_slot: int, T, max_range: float = 1.7976931348623157e308):
        """calc_fitness_score(target, source, T, max_range): (score, points counted)."""
        Tf = np.ascontiguousarray(T, np.float32)
        sc, n = C.c_double(), C.c_int()
        check(lib.lsd_loop_fitness(self.h, int(target_slot), int(source_slot), _ptr(Tf), max_range, C.byref(sc), C.byref(n)))
        return sc.value, n.value


def find_loop_candidates(poses, accum, keyframes, new_slot: int, last_edge_accum_distance: float = 0.0, params=None, **kw):
    """LoopDetector::find_candidates and the guesses of matching() (pure host, no device needed)."""
    p = params if params is not None else _loop_params(**kw)
    P, kf = _poses(poses), _slots(keyframes)
    acc = np.ascontiguousarray(accum, np.float64)
    if acc.size != P.shape[0] or not 0 <= new_slot < P.shape[0]:
        raise ValueError("one accum_distance and one pose per slot")
    cand = np.zeros(max(kf.size, 1), np.int32)
    G = np.zeros((max(kf.size, 1), 4, 4))
    n = C.c_int()
    check(lib.lsd_loop_find_candidates(C.byref(p), float(last_edge_accum_distance), _ptr(P), _ptr(acc), _ptr(kf), kf.size,
                                       int(new_slot), _ptr(cand), _ptr(G), cand.size, C.byref(n)))
    return cand[:n.value].copy(), G[:n.value].copy()


def loop_information_matrix(fitness_score: float) -> np.ndarray:
    """InformationMatrixCalculator::calc_information_matrix for a given fitness score (pure host)."""
    out = np.zeros((6, 6))
    lib.lsd_loop_information_matrix(float(fitness_score), _ptr(out))
    return out


def _galign_params(**kw) -> GalignParams:
    p = GalignParams()
    lib.lsd_galign_default_params(C.byref(p))
    for k, v in kw.items():
        if hasattr(p.reg, k) and not hasattr(p, k):
            setattr(p.reg, k, v)
        else:
            setattr(p, k, v)
    return p


class GlobalAligner:
    """The closure search of global_alignment (global_alignment.hpp:200-258) on the device: reference and new key frames
    are added once (clouds stay in device memory, addressed by slot); search() finds the ScanContext matches of each new
    key frame, aligns all (new, reference) pairs with batched FAST_VGICP and returns the closures that converged with a
    fitness score below 1.5.  Keyword arguments set lsd_galign_params_t fields or, by name, its matcher parameters."""

    def __init__(self, **kw):
        self.h = None
        self.params = _galign_params(**kw)
        self.h = C.c_void_p()
        check(lib.lsd_galign_create(C.byref(self.h), C.byref(self.params)))

    def close(self):
        if self.h:
            lib.lsd_galign_destroy(self.h)
        self.h = None

    __del__ = close

    def add_keyframe(self, pts, reference: bool) -> int:
        pts = _f32(pts)
        slot = C.c_int32()
        check(lib.lsd_galign_add_keyframe(self.h, _ptr(pts), pts.shape[0], int(bool(reference)), C.byref(slot)))
        return slot.value

    def search(self, new_slots) -> list[dict]:
        """Closures of the new key frames `new_slots`: ordered by new key frame, then ascending reference key frame."""
        ns = _slots(new_slots)
        cap = max(90 * ns.size, 1)   # at most 9 offsets x 10 ScanContext candidates per new key frame
        out = (GalignClosure * cap)()
        n = C.c_int()
        check(lib.lsd_galign_search(self.h, _ptr(ns), ns.size, out, cap, C.byref(n)))
        return [dict(ref_slot=c.ref_slot, new_slot=c.new_slot, relpose=np.array(c.relpose16, np.float32).reshape(4, 4),
                     score=c.score, sc_dist=c.sc_dist, sc_yaw=c.sc_yaw) for c in out[:n.value]]

    def matches(self) -> list[dict]:
        """Every pair the last search aligned, with its ScanContext match, LM outcome, score and gate decision."""
        n = C.c_int()
        check(lib.lsd_galign_last_matches(self.h, None, 0, C.byref(n)))
        out = (GalignMatch * max(n.value, 1))()
        check(lib.lsd_galign_last_matches(self.h, out, n.value, C.byref(n)))
        return [dict(new_slot=m.new_slot, ref_slot=m.ref_slot, sc_dist=m.sc_dist, sc_yaw=m.sc_yaw, converged=bool(m.converged),
                     iterations=m.iterations, score=m.score, accepted=bool(m.accepted)) for m in out[:n.value]]

    def set_max_batch_points(self, n: int):
        """Memory budget of the following searches (sum over a batch of new-cloud points x neighbours); no effect on results."""
        check(lib.lsd_galign_set_max_batch_points(self.h, int(n)))
        self.params.max_batch_points = int(n)

    def stats(self) -> dict:
        """Work of the last search: kernel launches of the matching, host round trips (cost rounds), batches."""
        ln, rd, nb = C.c_longlong(), C.c_int(), C.c_int()
        check(lib.lsd_galign_last_stats(self.h, C.byref(ln), C.byref(rd), C.byref(nb)))
        return dict(launches=ln.value, rounds=rd.value, batches=nb.value)

    def match(self, new_slot: int, ref_slots, guesses, serial: bool = False) -> dict:
        """FAST_VGICP of new_slot against each of ref_slots from guesses, batched or (serial) one pair at a time through
        the single-pair kernels on the same tables (parity tap and baseline)."""
        ref = _slots(ref_slots)
        n = ref.size
        G = np.ascontiguousarray(guesses, np.float64).reshape(n, 4, 4)
        T = np.zeros((n, 4, 4)); cv = np.zeros(n, np.int32); it = np.zeros(n, np.int32); fit = np.zeros(n)
        ln, rd = C.c_longlong(), C.c_int()
        check(lib.lsd_galign_match(self.h, int(new_slot), _ptr(ref), _ptr(G), n, int(bool(serial)), _ptr(T), _ptr(cv), _ptr(it),
                                   _ptr(fit), C.byref(ln), C.byref(rd)))
        logs = []
        for i in range(n):
            m = C.c_int()
            check(lib.lsd_galign_iteration_log(self.h, i, None, 0, C.byref(m)))
            lg = np.zeros((max(m.value, 1), 4))
            check(lib.lsd_galign_iteration_log(self.h, i, _ptr(lg), m.value, C.byref(m)))
            logs.append(lg[:m.value])
        return dict(final=T, converged=cv.astype(bool), iterations=it, fitness=fit, launches=ln.value, rounds=rd.value,
                    iteration_logs=logs)

    def cost(self, new_slot: int, ref_slot: int, T, update: bool = True, deriv: bool = True):
        """One VGICP cost evaluation of the pair through the batched kernel: (err, H, b, n_corr), as Matcher.cost."""
        T = np.ascontiguousarray(T, np.float64)
        H, b = np.zeros((6, 6)), np.zeros(6)
        e, nc = C.c_double(), C.c_int()
        check(lib.lsd_galign_cost(self.h, int(new_slot), int(ref_slot), _ptr(T), int(update), _ptr(H) if deriv else None,
                                  _ptr(b) if deriv else None, C.byref(e), C.byref(nc)))
        return e.value, H, b, nc.value


def _overlap_params(**kw) -> OverlapParams:
    p = OverlapParams()
    lib.lsd_overlap_default_params(C.byref(p))
    for k, v in kw.items():
        if k in ("coarse", "accurate"):          # dict of lsd_reg_params_t fields
            for kk, vv in v.items():
                if not hasattr(p.coarse, kk):
                    raise TypeError(f"unknown matcher parameter {kk}")
                setattr(getattr(p, k), kk, vv)
        elif hasattr(p, k):
            setattr(p, k, v)
        else:
            raise TypeError(f"unknown overlap-detector parameter {k}")
    return p


def _edges(a) -> np.ndarray:
    e = np.ascontiguousarray(a, np.int32).reshape(-1, 2) if len(a) else np.zeros((0, 2), np.int32)
    return np.ascontiguousarray(e)


class OverlapDetector:
    """OverlapDetector (overlap_merge.hpp) of map merging on the device: key frames of both maps are added once with their
    graph ids (clouds stay in device memory, addressed by slot); detect() finds the candidates of every new key frame of a
    fragment, prescreens and NDT-aligns all (new, candidate) pairs in batches, refines each new key frame's best
    candidate with GICP against the candidate accumulated with its graph neighbours and returns the overlaps."""

    def __init__(self, **kw):
        self.h = None
        self.params = _overlap_params(**kw)
        self.h = C.c_void_p()
        check(lib.lsd_overlap_create(C.byref(self.h), C.byref(self.params)))
        self.ids = []

    def close(self):
        if self.h:
            lib.lsd_overlap_destroy(self.h)
        self.h = None

    __del__ = close

    def add_keyframe(self, pts, kf_id: int) -> int:
        pts = _f32(pts)
        slot = C.c_int32()
        check(lib.lsd_overlap_add_keyframe(self.h, _ptr(pts), pts.shape[0], int(kf_id), C.byref(slot)))
        self.ids.append(int(kf_id))
        return slot.value

    def detect(self, poses, keyframes, new_keyframes, edges) -> list[dict]:
        """poses: mOdom of every slot [n_slots, 4, 4]; keyframes: the loaded map's slots (mKeyFrames order); new_keyframes:
        the fragment's slots; edges: graph edges as (prev id, next id) pairs.  One dict per overlap."""
        P, kf, nk, E = _poses(poses), _slots(keyframes), _slots(new_keyframes), _edges(edges)
        cap = max(nk.size, 1)
        out = (OverlapResult * cap)()
        n = C.c_int()
        check(lib.lsd_overlap_detect(self.h, _ptr(P), _ptr(kf), kf.size, _ptr(nk), nk.size, _ptr(E), E.shape[0], out, cap, C.byref(n)))
        return [dict(key1=r.key1, key2=r.key2, relpose=np.array(r.relpose16).reshape(4, 4), score=r.score,
                     coarse_score=r.coarse_score) for r in out[:n.value]]

    def reports(self) -> list[dict]:
        """What the last detect() decided for each new key frame (decision: OVERLAP_*)."""
        n = C.c_int()
        check(lib.lsd_overlap_last_reports(self.h, None, 0, C.byref(n)))
        out = (OverlapReport * max(n.value, 1))()
        check(lib.lsd_overlap_last_reports(self.h, out, n.value, C.byref(n)))
        return [{k: getattr(r, k) for k, _ in OverlapReport._fields_} for r in out[:n.value]]

    def stats(self) -> dict:
        """Work of the last detect(): kernel launches, host round trips of the NDT stage; target table sets owned / held."""
        ln, rd, tb, th = C.c_longlong(), C.c_int(), C.c_int(), C.c_int()
        check(lib.lsd_overlap_last_stats(self.h, C.byref(ln), C.byref(rd), C.byref(tb), C.byref(th)))
        return dict(launches=ln.value, rounds=rd.value, target_buffers=tb.value, targets_held=th.value)

    def release_targets(self):
        """Hand back the tables fitness() and match() built and kept (detect() releases its own when it returns)."""
        check(lib.lsd_overlap_release_targets(self.h))

    def find_candidates(self, poses, keyframes, new_slot: int, edges) -> np.ndarray:
        return overlap_find_candidates(poses, self.ids, keyframes, new_slot, edges, params=self.params)

    def fitness(self, target_slot: int, source_slot: int, T, max_range: float) -> dict:
        """calc_fitness_score(target, source, T, max_range) of the reference's merge (filtered clouds)."""
        Tf = np.ascontiguousarray(T, np.float32)
        sc, ratio = C.c_double(), C.c_double()
        nr, nf, inc = C.c_int(), C.c_int(), C.c_int()
        check(lib.lsd_overlap_fitness(self.h, int(target_slot), int(source_slot), _ptr(Tf), float(max_range), C.byref(sc), C.byref(ratio),
                                      C.byref(nr), C.byref(nf), C.byref(inc)))
        return dict(score=sc.value, inlier_ratio=ratio.value, n_counted=nr.value, n_filtered=nf.value, target_incomplete=bool(inc.value))

    def match(self, new_slots, cand_slots, guesses, serial: bool = False) -> dict:
        """The coarse stage alone for an explicit pair list, batched or (serial) one pair at a time through lsd_reg's
        single-pair kernels on the same tables (parity tap and baseline)."""
        ns, cs = _slots(new_slots), _slots(cand_slots)
        n = cs.size
        G = np.ascontiguousarray(guesses, np.float64).reshape(n, 4, 4)
        T = np.zeros((n, 4, 4)); cv = np.zeros(n, np.int32); it = np.zeros(n, np.int32); fit = np.zeros(n)
        ln, rd = C.c_longlong(), C.c_int()
        check(lib.lsd_overlap_match(self.h, _ptr(ns), _ptr(cs), _ptr(G), n, int(bool(serial)), _ptr(T), _ptr(cv), _ptr(it), _ptr(fit), C.byref(ln), C.byref(rd)))
        logs = []
        for i in range(n):
            m = C.c_int()
            check(lib.lsd_overlap_iteration_log(self.h, i, None, 0, C.byref(m)))
            lg = np.zeros((max(m.value, 1), 4))
            check(lib.lsd_overlap_iteration_log(self.h, i, _ptr(lg), m.value, C.byref(m)))
            logs.append(lg[:m.value])
        return dict(final=T, converged=cv.astype(bool), iterations=it, fitness=fit, launches=ln.value, rounds=rd.value,
                    iteration_logs=logs)


def overlap_find_candidates(poses, ids, keyframes, new_slot: int, edges, params=None, **kw) -> np.ndarray:
    """OverlapDetector::find_candidates (pure host, no device needed): candidate slots in 10-NN order."""
    p = params if params is not None else _overlap_params(**kw)
    P, kf, E = _poses(poses), _slots(keyframes), _edges(edges)
    idv = np.ascontiguousarray(ids, np.int32)
    if idv.size != P.shape[0]:
        raise ValueError("one id and one pose per slot")
    cand = np.zeros(max(kf.size, 1), np.int32)
    n = C.c_int()
    check(lib.lsd_overlap_find_candidates(C.byref(p), _ptr(P), _ptr(idv), P.shape[0], _ptr(kf), kf.size, _ptr(E), E.shape[0], int(new_slot),
                                          _ptr(cand), cand.size, C.byref(n)))
    return cand[:n.value].copy()


def overlap_guess(T_new, T_cand) -> np.ndarray:
    """(new.inverse() * cand).matrix().cast<float>() of the reference's prescreen and NDT guess (pure host)."""
    a, b = np.ascontiguousarray(T_new, np.float64), np.ascontiguousarray(T_cand, np.float64)
    out = np.zeros((4, 4), np.float32)
    lib.lsd_overlap_guess(_ptr(a), _ptr(b), _ptr(out))
    return out


def overlap_finetune_guess(ndt_final) -> np.ndarray:
    """Eigen::Isometry3f(ndt_final).inverse().matrix() in float (pure host)."""
    a = np.ascontiguousarray(ndt_final, np.float32)
    out = np.zeros((4, 4), np.float32)
    lib.lsd_overlap_finetune_guess(_ptr(a), _ptr(out))
    return out


def galign_merge_candidates(cand_idx, cand_dist, cand_shift, n_cand, dist_thres: float = 0.30):
    """global_alignment.hpp:215-227 on lsd_sc_query output ([n_off, 10] each, n_cand [n_off]): the matches below
    dist_thres merged per database index (pure host).  Returns (idx [m], sc_dist float32 [m], sc_yaw float32 [m])."""
    idx = np.ascontiguousarray(cand_idx, np.int32).reshape(-1, 10)
    n_off = idx.shape[0]
    dist = np.ascontiguousarray(cand_dist, np.float64).reshape(n_off, 10)
    sh = np.ascontiguousarray(cand_shift, np.int32).reshape(n_off, 10)
    nc = np.ascontiguousarray(n_cand, np.int32).reshape(n_off)
    cap = max(n_off * 10, 1)
    oi, od, oy = np.zeros(cap, np.int32), np.zeros(cap, np.float32), np.zeros(cap, np.float32)
    n = C.c_int()
    check(lib.lsd_galign_merge_candidates(_ptr(idx), _ptr(dist), _ptr(sh), _ptr(nc), n_off, float(dist_thres), _ptr(oi), _ptr(od),
                                          _ptr(oy), cap, C.byref(n)))
    return oi[:n.value].copy(), od[:n.value].copy(), oy[:n.value].copy()


def floor_params(preset: int = FLOOR_MAPPING, **kw) -> FloorParams:
    p = FloorParams()
    lib.lsd_floor_default_params(C.byref(p), int(preset))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(f"lsd_floor_params_t has no field {k}")
        setattr(p, k, v)
    return p


class FloorDetector:
    """Floor detection on the device (FloorDetectionNodelet::detect and the two detect_ground copies): height clip,
    k = 10 normal filter and RANSAC plane fit, one frame per detect().  preset: FLOOR_MAPPING (with the prefilter),
    FLOOR_GROUND or FLOOR_RENDER; keyword arguments set lsd_floor_params_t fields."""

    def __init__(self, preset: int = FLOOR_MAPPING, **kw):
        self.h = None
        self.params = floor_params(preset, **kw)
        self.h = C.c_void_p()
        check(lib.lsd_floor_create(C.byref(self.h), C.byref(self.params)))

    def close(self):
        if self.h:
            lib.lsd_floor_destroy(self.h)
        self.h = None

    __del__ = close

    def detect(self, pts) -> dict:
        """One frame: [n,4] float32 (numpy: host input; torch CUDA tensor: device input).  Returns the result fields;
        coeffs is float32[4] (upward normal when found)."""
        r = FloorResult()
        if isinstance(pts, np.ndarray):
            a = _f32(pts)
            check(lib.lsd_floor_detect(self.h, _ptr(a), a.shape[0], C.byref(r)))
        else:
            if str(pts.dtype) != "torch.float32" or pts.dim() != 2 or pts.shape[1] != 4 or not pts.is_contiguous():
                raise ValueError("device points must be a contiguous float32 [n,4] tensor")
            check(lib.lsd_floor_detect_dev(self.h, pts.data_ptr(), pts.shape[0], C.byref(r)))
        out = {k: getattr(r, k) for k, _ in r._fields_}
        out["coeffs"] = np.array(r.coeffs, np.float32)
        out["found"] = bool(r.found)
        return out

    def cloud(self, stage: str) -> np.ndarray:
        """The cloud of a stage of the last detect: 'prefiltered', 'clipped', 'candidates' or 'inliers'."""
        s = FLOOR_STAGES[stage]
        n = C.c_int()
        check(lib.lsd_floor_get_cloud(self.h, s, None, 0, C.byref(n)))
        out = np.zeros((max(n.value, 1), 4), np.float32)
        check(lib.lsd_floor_get_cloud(self.h, s, _ptr(out), n.value, C.byref(n)))
        return out[:n.value]

    def normals(self):
        """(normal4 [m,4] = nx, ny, nz, curvature; cov6 [m,6] = xx, xy, xz, yy, yz, zz) per clipped point of the last detect."""
        n = C.c_int()
        check(lib.lsd_floor_get_normals(self.h, None, None, 0, C.byref(n)))
        nr, cv = np.zeros((max(n.value, 1), 4), np.float32), np.zeros((max(n.value, 1), 6), np.float32)
        check(lib.lsd_floor_get_normals(self.h, _ptr(nr), _ptr(cv), n.value, C.byref(n)))
        return nr[:n.value], cv[:n.value]

    def samples(self):
        """The hypotheses RANSAC drew in the last detect, in draw order: (idx [m,3], flags [m], counts [m])."""
        n = C.c_int()
        check(lib.lsd_floor_last_samples(self.h, None, None, None, 0, C.byref(n)))
        m = max(n.value, 1)
        idx, fl, cn = np.zeros((m, 3), np.int32), np.zeros(m, np.int32), np.zeros(m, np.int32)
        check(lib.lsd_floor_last_samples(self.h, _ptr(idx), _ptr(fl), _ptr(cn), n.value, C.byref(n)))
        return idx[:n.value], fl[:n.value], cn[:n.value]


def ransac_replay(counts, flags, n_points: int, probability: float = 0.99, max_iterations: int = 10000) -> dict:
    """RandomSampleConsensus::computeModel's stop rule on hypotheses in draw order (pure host).  consumed = -1: the loop
    had not ended after the given hypotheses."""
    cn = np.ascontiguousarray(counts, np.int32).ravel()
    fl = np.ascontiguousarray(flags, np.int32).ravel()
    if cn.size != fl.size:
        raise ValueError("counts and flags differ in length")
    c, b, it, sk = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    check(lib.lsd_ransac_replay(_ptr(cn), _ptr(fl), cn.size, int(n_points), float(probability), int(max_iterations), C.byref(c),
                                C.byref(b), C.byref(it), C.byref(sk)))
    return dict(consumed=c.value, best=b.value, iterations=it.value, skipped=sk.value)


def eskf_update_table(state, P, HTH, HTh, n_eff, R=0.001, max_iterations=4, eps=0.001, literal=False, converge_log=None):
    """Host-only filter run with a tabulated measurement model (include/lsdreg.h lsd_eskf_update_table).
    converge_log: optional int32[16] receiving the converge flag of every evaluation."""
    state = np.array(state, np.float64)
    P = np.array(P, np.float64)
    HTH = np.ascontiguousarray(HTH, np.float64).reshape(-1, 36)
    HTh = np.ascontiguousarray(HTh, np.float64).reshape(-1, 6)
    n_eff = np.ascontiguousarray(n_eff, np.int32)
    ev = lib.lsd_eskf_update_table(_ptr(state), _ptr(P), _ptr(HTH), _ptr(HTh), _ptr(n_eff), HTH.shape[0], R, max_iterations,
                                   eps, int(literal), None if converge_log is None else _ptr(converge_log))
    return state, P, ev


IMU_INITIALIZING = 4
LOCALMAP_NONE = 5


class LocalMap:
    """Localization::runUpdateLocalMap's map assembly (localization.cpp:303-373) on device-resident key frames."""

    def __init__(self, resolution: float = 0.5, key_frame_distance: float = 1.0):
        self.h = C.c_void_p()
        check(lib.lsd_localmap_create(C.byref(self.h), resolution, key_frame_distance))

    def close(self):
        if getattr(self, "h", None):
            lib.lsd_localmap_destroy(self.h)
        self.h = None

    __del__ = close

    def add_keyframe(self, pts_map_frame, position):
        pts = _f32(pts_map_frame)
        pos = np.ascontiguousarray(position, np.float64)
        check(lib.lsd_localmap_add_keyframe(self.h, _ptr(pts), pts.shape[0], _ptr(pos)))

    def update(self, pose_xyz):
        """-> (status, n_points, n_keyframes_in_radius, nearest_dist)"""
        p = np.ascontiguousarray(pose_xyz, np.float64)
        n, k, d = C.c_int(), C.c_int(), C.c_double()
        st = check(lib.lsd_localmap_update(self.h, _ptr(p), C.byref(n), C.byref(k), C.byref(d)))
        return st, n.value, k.value, d.value

    def cloud(self) -> np.ndarray:
        n = C.c_int()
        check(lib.lsd_localmap_get(self.h, None, 0, C.byref(n)))
        out = np.empty((n.value, 4), np.float32)
        check(lib.lsd_localmap_get(self.h, _ptr(out), n.value, C.byref(n)))
        return out

    def cloud_dev(self):
        p, n = C.c_void_p(), C.c_int()
        check(lib.lsd_localmap_get_dev(self.h, C.byref(p), C.byref(n)))
        return p.value, n.value


class FastLio:
    """The reference's LIO seam (fastlio.cpp:9-16: fastlio_init / _imu_enqueue / _ins_enqueue / _pcl_enqueue / fastlio_main /
    _odometry / _state / _is_init) on lsd_fastlio_*.  Same feeding protocol as oracle/fastlio.py's RefFastLio."""

    def __init__(self, ext_R=None, ext_t=None, filter_num=1, max_point_num=-1, scan_period=0.1, undistort=True,
                 map_log2_lines=None, max_scan_points=None):
        R = np.ascontiguousarray(np.eye(3) if ext_R is None else ext_R, np.float64).reshape(-1)
        t = np.ascontiguousarray(np.zeros(3) if ext_t is None else ext_t, np.float64)
        self.h = C.c_void_p()
        check(lib.lsd_fastlio_create(C.byref(self.h), _ptr(t), _ptr(R), filter_num, max_point_num, scan_period, int(undistort)))
        if map_log2_lines is not None or max_scan_points is not None:
            check(lib.lsd_fastlio_set_capacity(self.h, map_log2_lines or 22, max_scan_points or 262144))

    def close(self):
        if getattr(self, "h", None):
            lib.lsd_fastlio_destroy(self.h)
        self.h = None

    __del__ = close

    def push_imu(self, stamp, gyr, acc_g):
        """acc in units of g like the rest of the package; the entry point takes m/s^2 (fastlio_imu_enqueue divides by 9.81)."""
        g = np.ascontiguousarray(gyr, np.float64)
        a = np.ascontiguousarray(acc_g, np.float64) * 9.81
        check(lib.lsd_fastlio_imu_enqueue(self.h, float(stamp), _ptr(g), _ptr(a)))

    def push_ins(self, timestamp_us, vel_enu, heading_deg, pitch_deg, roll_deg, rtk_valid=True, is_wheel=False):
        v = np.ascontiguousarray(vel_enu, np.float64)
        check(lib.lsd_fastlio_ins_enqueue(self.h, int(rtk_valid), int(is_wheel), int(timestamp_us), _ptr(v), heading_deg, pitch_deg, roll_deg))

    def push_scan(self, xyzi, stamp_us, header_stamp_us):
        xyzi = _f32(xyzi)
        st = np.ascontiguousarray(stamp_us, np.uint32)
        check(lib.lsd_fastlio_pcl_enqueue(self.h, _ptr(xyzi), _ptr(st), xyzi.shape[0], int(header_stamp_us)))

    def step(self) -> bool:
        """fastlio_main()"""
        return bool(check(lib.lsd_fastlio_main(self.h)))

    def last(self):
        st, info = C.c_int(), LioInfo()
        check(lib.lsd_fastlio_last(self.h, C.byref(st), C.byref(info)))
        return dict(info.as_dict(), status=st.value)

    def filter(self):
        x, P = np.zeros(26), np.zeros((23, 23))
        check(lib.lsd_fastlio_get_filter(self.h, _ptr(x), _ptr(P)))
        return x, P

    def odometry(self):
        a, b = np.zeros((4, 4)), np.zeros((4, 4))
        check(lib.lsd_fastlio_odometry(self.h, _ptr(a), _ptr(b)))
        return a, b

    def state(self) -> np.ndarray:
        out = np.zeros(20)
        check(lib.lsd_fastlio_state(self.h, _ptr(out)))
        return out

    @property
    def initialised(self) -> bool:
        return bool(lib.lsd_fastlio_is_init(self.h))

    def lio_handle(self):
        return lib.lsd_fastlio_lio(self.h)

    def pop_package(self, cap_points=400000, cap_imu=4096):
        """Parity tap (host only): sync_packages alone -> dict or None."""
        beg, end, n, ni, hi = C.c_double(), C.c_double(), C.c_int(), C.c_int(), C.c_int()
        xyzi, t = np.zeros((cap_points, 4), np.float32), np.zeros(cap_points, np.float32)
        imu, iv = np.zeros((cap_imu, 7)), np.zeros(3)
        r = check(lib.lsd_fastlio_pop_package(self.h, C.byref(beg), C.byref(end), C.byref(n), _ptr(xyzi), _ptr(t), cap_points, C.byref(ni),
                                              _ptr(imu), cap_imu, C.byref(hi), _ptr(iv)))
        if not r:
            return None
        return dict(lidar_beg_time=beg.value, lidar_end_time=end.value, points=xyzi[:n.value].copy(), time_ms=t[:n.value].copy(),
                    imu=imu[:ni.value].copy(), ins_vel=iv.copy() if hi.value else None)


class ScanContext:
    """SCManager (slam/common/Scancontext/Scancontext.cpp) on the device: descriptors, database, retrieval.
    Descriptors are [60, 20] (sector, ring) float64 arrays = Eigen's column-major 20 x 60 MatrixXd."""

    MAX_QUERIES, CANDIDATES = 64, 10
    SEARCH_TRANS = [(0, 0), (-4, 0), (4, 0), (0, -4), (0, 4), (-4, -4), (-4, 4), (4, -4), (4, 4)]   # global_localization.cpp:390-392

    def __init__(self, db_capacity: int = 16384, dist_thres: float = 0.2):
        self.h = C.c_void_p()
        self.dist_thres = dist_thres   # SC_DIST_THRES
        check(lib.lsd_sc_create(C.byref(self.h), db_capacity))

    def close(self):
        if getattr(self, "h", None):
            lib.lsd_sc_destroy(self.h)
        self.h = None

    __del__ = close

    def make(self, pts, offsets=None, dev: bool = False):
        """makeScancontext + keys for every offset -> (desc [n_off,60,20], ringkey [n_off,20], sectorkey [n_off,60])."""
        off = np.ascontiguousarray(np.zeros((1, 2)) if offsets is None else offsets, np.float64).reshape(-1, 2)
        k = off.shape[0]
        desc, rk, sk = np.empty((k, 60, 20)), np.empty((k, 20)), np.empty((k, 60))
        if dev:
            check(lib.lsd_sc_make_dev(self.h, _ptr(pts), pts.shape[0], _ptr(off), k, _ptr(desc), _ptr(rk), _ptr(sk)))
        else:
            pts = _f32(pts)
            check(lib.lsd_sc_make(self.h, _ptr(pts), pts.shape[0], _ptr(off), k, _ptr(desc), _ptr(rk), _ptr(sk)))
        return desc, rk, sk

    def db_clear(self):
        check(lib.lsd_sc_db_clear(self.h))

    def db_add(self, descs):
        d = np.ascontiguousarray(descs, np.float64).reshape(-1, 1200)
        check(lib.lsd_sc_db_add(self.h, _ptr(d), d.shape[0]))

    def db_add_made(self, slot: int = 0):
        check(lib.lsd_sc_db_add_made(self.h, slot))

    def db_size(self) -> int:
        n = C.c_int()
        check(lib.lsd_sc_db_size(self.h, C.byref(n)))
        return n.value

    def query(self, descs=None, nq: int | None = None):
        """-> (cand_idx [nq,10], cand_dist [nq,10], cand_shift [nq,10], n_cand [nq]); descs None = the last make()."""
        d = None
        if descs is not None:
            d = np.ascontiguousarray(descs, np.float64).reshape(-1, 1200)
            nq = d.shape[0]
        idx, dist = np.empty((nq, 10), np.int32), np.empty((nq, 10))
        sh, nc = np.empty((nq, 10), np.int32), np.empty(nq, np.int32)
        check(lib.lsd_sc_query(self.h, _ptr(d) if d is not None else None, nq, _ptr(idx), _ptr(dist), _ptr(sh), _ptr(nc)))
        return idx, dist, sh, nc

    def distance(self, a, b):
        """distanceBtnScanContext for pairs -> (dist [n], shift [n])."""
        a = np.ascontiguousarray(a, np.float64).reshape(-1, 1200)
        b = np.ascontiguousarray(b, np.float64).reshape(-1, 1200)
        n = a.shape[0]
        dist, sh = np.empty(n), np.empty(n, np.int32)
        check(lib.lsd_sc_distance(self.h, _ptr(a), _ptr(b), n, _ptr(dist), _ptr(sh)))
        return dist, sh

    def detect_closest(self, slot: int = 0):
        """detectClosestMatch for query slot `slot` -> (loop id or -1, yaw rad, score); score 1.0 on an empty database
        (what globalSearch passes in, global_localization.cpp:397)."""
        lid, yaw, score = C.c_int32(), C.c_float(), C.c_double(1.0)
        check(lib.lsd_sc_detect_closest(self.h, slot, self.dist_thres, C.byref(lid), C.byref(yaw), C.byref(score)))
        return lid.value, yaw.value, score.value

    def detect_candidates(self, slot: int = 0):
        idx, yaw, dist, n = np.empty(10, np.int32), np.empty(10, np.float32), np.empty(10, np.float32), C.c_int32()
        check(lib.lsd_sc_detect_candidates(self.h, slot, self.dist_thres, _ptr(idx), _ptr(yaw), _ptr(dist), C.byref(n)))
        return [(int(idx[i]), float(yaw[i]), float(dist[i])) for i in range(n.value)]


def keyframe_filter(pts, radius: float = 1.0, min_neighbors: int = 3, min_range: float = 0.0, max_range: float = 1e9):
    """RadiusOutlierRemoval + pointsDistanceFilter of a new key frame (slam.cpp:398-410); order preserving."""
    pts = _f32(pts)
    out = np.empty_like(pts)
    n = C.c_int()
    check(lib.lsd_keyframe_filter(_ptr(pts), pts.shape[0], radius, min_neighbors, min_range, max_range, _ptr(out), C.byref(n)))
    return out[:n.value].copy()


def keyframe_save(directory: str, stamp_us: int, kf_id: int, pts, pose):
    """dump_keyframe / KeyFrame::save: <directory>/cloud.pcd (binary PCD, intensity x 255) and <directory>/data."""
    pts = _f32(pts)
    pose = np.ascontiguousarray(pose, np.float64).reshape(4, 4)
    check(lib.lsd_keyframe_save(os.fsencode(directory), int(stamp_us), int(kf_id), _ptr(pts), pts.shape[0], _ptr(pose)))


def keyframe_load(directory: str):
    """KeyFrame(id, directory, True).loadOdom() + loadPcd(): -> (stamp_us, id, pose [4,4], points [n,4] with intensity / 255)."""
    stamp, kid, n = C.c_uint64(), C.c_int64(), C.c_int()
    pose = np.zeros((4, 4))
    check(lib.lsd_keyframe_load(os.fsencode(directory), C.byref(stamp), C.byref(kid), _ptr(pose), None, 0, C.byref(n)))
    pts = np.zeros((max(n.value, 1), 4), np.float32)
    check(lib.lsd_keyframe_load(os.fsencode(directory), C.byref(stamp), C.byref(kid), _ptr(pose), _ptr(pts), pts.shape[0], C.byref(n)))
    return stamp.value, kid.value, pose, pts[:n.value]


def eskf_predict(state, P, dt, Q, acc, gyro):
    """esekf::predict on the host (no GPU): returns (state, P) after one step."""
    state = np.ascontiguousarray(state, np.float64).copy()
    P = np.ascontiguousarray(P, np.float64).copy()
    Q = np.ascontiguousarray(Q, np.float64); acc = np.ascontiguousarray(acc, np.float64); gyro = np.ascontiguousarray(gyro, np.float64)
    check(lib.lsd_eskf_predict(_ptr(state), _ptr(P), float(dt), _ptr(Q), _ptr(acc), _ptr(gyro)))
    return state, P


class ImuProcess:
    """ImuProcess (IMU_Processing.hpp): IMU initialisation, forward propagation, undistortion."""

    def __init__(self, ext_R=None, ext_t=None, **kw):
        self.h = None
        self.params = ImuParams()
        lib.lsd_imu_default_params(C.byref(self.params))
        if ext_R is not None:
            self.params.ext_R[:] = list(np.asarray(ext_R, np.float64).reshape(9))
        if ext_t is not None:
            self.params.ext_t[:] = list(np.asarray(ext_t, np.float64).reshape(3))
        for k, v in kw.items():
            if not hasattr(self.params, k):
                raise TypeError(f"unknown ImuProcess parameter {k}")
            setattr(self.params, k, v)
        self.h = C.c_void_p()
        check(lib.lsd_imu_create(C.byref(self.h), C.byref(self.params)))

    def close(self):
        if self.h:
            lib.lsd_imu_destroy(self.h)
        self.h = None

    __del__ = close

    def is_init(self) -> bool:
        f = C.c_int()
        check(lib.lsd_imu_is_init(self.h, C.byref(f)))
        return bool(f.value)

    def process(self, imu, beg, end, points, time_ms, state, P, ins_vel=None):
        """-> (status, state, P, n_undistorted).  status IMU_INITIALIZING until the IMU is initialised.
        points/time_ms: numpy (host path) or CUDA torch tensors (device path)."""
        imu = np.ascontiguousarray(imu, np.float64).reshape(-1, 7)
        state = np.ascontiguousarray(state, np.float64).copy()
        P = np.ascontiguousarray(P, np.float64).copy()
        iv = None if ins_vel is None else np.ascontiguousarray(ins_vel, np.float64)
        n = C.c_int()
        if isinstance(points, np.ndarray):
            points = _f32(points)
            time_ms = np.ascontiguousarray(time_ms, np.float32)
            fn = lib.lsd_imu_process
        else:
            fn = lib.lsd_imu_process_dev
        st = check(fn(self.h, _ptr(imu), imu.shape[0], None if iv is None else _ptr(iv), float(beg), float(end), _ptr(points),
                      _ptr(time_ms), points.shape[0], _ptr(state), _ptr(P), C.byref(n)))
        return st, state, P, n.value

    def cloud(self) -> np.ndarray:
        n = C.c_int()
        check(lib.lsd_imu_get_cloud(self.h, None, 0, C.byref(n)))
        out = np.empty((n.value, 4), np.float32)
        check(lib.lsd_imu_get_cloud(self.h, _ptr(out), n.value, C.byref(n)))
        return out

    def cloud_dev(self):
        """(device pointer, n, cudaStream_t) of the undistorted cloud."""
        p, n, st = C.c_void_p(), C.c_int(), C.c_void_p()
        check(lib.lsd_imu_get_cloud_dev(self.h, C.byref(p), C.byref(n), C.byref(st)))
        return p.value, n.value, st.value or 0

    def poses(self) -> np.ndarray:
        n = C.c_int()
        check(lib.lsd_imu_get_poses(self.h, None, 0, C.byref(n)))
        out = np.empty((n.value, 22), np.float64)
        check(lib.lsd_imu_get_poses(self.h, _ptr(out), n.value, C.byref(n)))
        return out


class LioFrontend:
    """Per-scan LIO pass (fastlio_main body): downsample -> iterated ESKF update -> map_incremental."""

    def __init__(self, **kw):
        self.params = LioParams()
        lib.lsd_lio_default_params(C.byref(self.params))
        for k, v in kw.items():
            if not hasattr(self.params, k):
                raise TypeError(f"unknown LIO parameter {k}")
            setattr(self.params, k, v)
        self.h = C.c_void_p()
        check(lib.lsd_lio_create(C.byref(self.h), C.byref(self.params)))
        self.map = HashVoxelMap(_borrow=lib.lsd_lio_map(self.h))
        self.n_down = 0

    def close(self):
        if self.h:
            lib.lsd_lio_destroy(self.h)
        self.h = None

    __del__ = close

    def set_nearby(self, stencil: int):
        check(lib.lsd_lio_set_nearby(self.h, stencil))

    def set_next_id(self, i: int):
        check(lib.lsd_lio_set_next_id(self.h, i))

    def set_ekf_inited(self, flag: bool):
        check(lib.lsd_lio_set_ekf_inited(self.h, int(flag)))

    def set_stale_rows(self, flag: bool):
        """Keep Nearest_Points[i] when a search finds nothing, as the reference does (include/lsdreg.h)."""
        check(lib.lsd_lio_set_stale_rows(self.h, int(flag)))

    def set_reference_order(self, flag: bool):
        """Nearest_Points rows in the order IVox::GetClosestPoint returns them (include/lsdreg.h)."""
        check(lib.lsd_lio_set_reference_order(self.h, int(flag)))

    def reference_order_fallbacks(self) -> int:
        c = C.c_uint()
        check(lib.lsd_lio_reference_order_fallbacks(self.h, C.byref(c)))
        return c.value

    def set_knn_shape(self, shape: int):
        """0/1 = one warp per scan point, 3 = flat (include/lsdreg.h::lsd_lio_set_knn_shape)."""
        check(lib.lsd_lio_set_knn_shape(self.h, int(shape)))

    def set_pipeline(self, flag: bool):
        """Voxel grid of a prefetched scan on the copy stream while the previous scan iterates (include/lsdreg.h::lsd_lio_set_pipeline)."""
        check(lib.lsd_lio_set_pipeline(self.h, int(flag)))

    def pipeline_stats(self):
        a, b = C.c_longlong(), C.c_longlong()
        check(lib.lsd_lio_pipeline_stats(self.h, C.byref(a), C.byref(b)))
        return dict(issued=a.value, adopted=b.value)

    def set_pdl(self, flag: bool):
        """Programmatic dependent launch for the scan's kernel chain (include/lsdreg.h::lsd_lio_set_pdl)."""
        check(lib.lsd_lio_set_pdl(self.h, int(flag)))

    SHARD_BLOB_BYTES = 192

    def shard_export(self, rank: int, world: int, tile_cells: int = 32, reach_cells: int = 1) -> np.ndarray:
        blob = np.zeros(self.SHARD_BLOB_BYTES, np.uint8)
        check(lib.lsd_lio_shard_export(self.h, rank, world, tile_cells, reach_cells, _ptr(blob)))
        return blob

    def shard_connect(self, blobs: np.ndarray):
        blobs = np.ascontiguousarray(blobs, np.uint8)
        check(lib.lsd_lio_shard_connect(self.h, _ptr(blobs)))

    def shard_exchange_stats(self):
        us, n = C.c_double(), C.c_longlong()
        check(lib.lsd_lio_shard_exchange_stats(self.h, C.byref(us), C.byref(n)))
        return dict(mean_us=us.value, evaluations=n.value)

    def sync(self):
        """Drain the handle's stream -> (gpu_ms, n_added) of the last scan."""
        ms, na = C.c_double(), C.c_int()
        check(lib.lsd_lio_sync(self.h, C.byref(ms), C.byref(na)))
        return ms.value, na.value

    def set_profile(self, on: bool):
        check(lib.lsd_lio_set_profile(self.h, int(on)))

    def get_profile(self):
        ms = np.zeros(4)
        cnt = np.zeros(4, np.int64)
        check(lib.lsd_lio_get_profile(self.h, _ptr(ms), _ptr(cnt)))
        names = ("hmodel_search", "hmodel_reuse", "voxelgrid", "map_incremental")
        return {n: dict(ms=float(ms[i]), count=int(cnt[i])) for i, n in enumerate(names)}

    def load_scan(self, scan, downsample: bool = True) -> int:
        n_down = C.c_int()
        if isinstance(scan, np.ndarray):
            scan = _f32(scan)
            check(lib.lsd_lio_load_scan(self.h, _ptr(scan), scan.shape[0], int(downsample), C.byref(n_down)))
        else:
            check(lib.lsd_lio_load_scan_dev(self.h, _ptr(scan), scan.shape[0], int(downsample), C.byref(n_down)))
        self.n_down = n_down.value
        return n_down.value

    def get_down(self) -> np.ndarray:
        out = np.empty((max(self.n_down, 1), 4), np.float32)
        n = C.c_int()
        check(lib.lsd_lio_get_down(self.h, _ptr(out), out.shape[0], C.byref(n)))
        return out[:n.value].copy()

    def linearize(self, state: np.ndarray, search: bool = True):
        state = np.ascontiguousarray(state, np.float64)
        HTH, HTh = np.zeros((6, 6)), np.zeros(6)
        rs, ne, dg = C.c_double(), C.c_int(), C.c_int()
        st = check(lib.lsd_lio_linearize(self.h, _ptr(state), int(search), _ptr(HTH), _ptr(HTh), C.byref(rs),
                                         C.byref(ne), C.byref(dg)))
        return dict(status=st, HTH=HTH, HTh=HTh, res_sum=rs.value, n_eff=ne.value, degenerate=dg.value)

    def get_matches(self):
        n = self.n_down
        idx = np.empty((n, 5), np.int32)
        xyz = np.empty((n, 5, 3), np.float32)
        cnt = np.empty(n, np.int32)
        sel = np.empty(n, np.uint8)
        plane = np.empty((n, 4), np.float32)
        world = np.empty((n, 4), np.float32)
        check(lib.lsd_lio_get_matches(self.h, _ptr(idx), _ptr(xyz), _ptr(cnt), _ptr(sel), _ptr(plane), _ptr(world)))
        return dict(idx=idx, xyz=xyz, cnt=cnt, selected=sel, plane=plane, world=world)

    def get_map_flags(self):
        """-> (flags [n] uint8, travel_distance): the last map_incremental's decision per downsampled point (0 = not added,
        1 = PointToAdd, 2 = PointNoNeedDownsample) and the travel distance handed to the map's LRU."""
        n, d = C.c_int(), C.c_double()
        check(lib.lsd_lio_get_map_flags(self.h, None, 0, C.byref(n), C.byref(d)))
        flags = np.empty(max(n.value, 1), np.uint8)
        check(lib.lsd_lio_get_map_flags(self.h, _ptr(flags), n.value, C.byref(n), C.byref(d)))
        return flags[:n.value], d.value

    def update(self, state: np.ndarray, P: np.ndarray):
        state = np.array(state, np.float64)
        P = np.array(P, np.float64)
        info = LioInfo()
        st = check(lib.lsd_lio_update(self.h, _ptr(state), _ptr(P), C.byref(info)))
        self.n_down = info.n_down
        return state, P, dict(info.as_dict(), status=st)

    def map_incremental(self, state: np.ndarray) -> int:
        state = np.ascontiguousarray(state, np.float64)
        n = C.c_int()
        check(lib.lsd_lio_map_incremental(self.h, _ptr(state), C.byref(n)))
        return n.value

    def prefetch(self, scan):
        """Start the H2D copy of the NEXT scan (host numpy / pinned torch tensor); the following scan() with the
        same buffer uses the staged copy.  Keep the buffer alive and unchanged until then."""
        if isinstance(scan, np.ndarray):
            if scan.dtype != np.float32 or not scan.flags.c_contiguous:
                raise ValueError("prefetch needs the exact float32 C-contiguous buffer later passed to scan()")
        elif getattr(scan, "is_cuda", False):      # device-resident scan: only the pipelined voxel grid has work to do ahead
            check(lib.lsd_lio_prefetch_dev(self.h, _ptr(scan), scan.shape[0]))
            return
        check(lib.lsd_lio_prefetch(self.h, _ptr(scan), scan.shape[0]))

    def scan_into(self, scan, state: np.ndarray, P: np.ndarray, info: "LioInfo") -> int:
        """scan() without the per-call allocations: `state` (float64 state vector) and `P` (float64[23,23], C order) are updated in
        place, `info` is a caller-owned LioInfo, `scan` must already be float32 [n,4] C-contiguous (numpy, pinned or CUDA
        torch tensor).  Returns the status code (raises like scan()).  For callers that register thousands of scans per
        second, where building two arrays and a dict per call is a tenth of the step."""
        fn = lib.lsd_lio_scan_dev if getattr(scan, "is_cuda", False) else lib.lsd_lio_scan
        st = fn(self.h, _ptr(scan), scan.shape[0], state.ctypes.data, P.ctypes.data, C.byref(info))
        if st < 0:
            check(st)
        self.n_down = info.n_down
        return st

    def scan(self, scan, state: np.ndarray, P: np.ndarray):
        """Whole pass.  `scan`: numpy [n,4] (host pointer, H2D inside) or CUDA torch tensor (device)."""
        state = np.array(state, np.float64)
        P = np.array(P, np.float64)
        info = LioInfo()
        if isinstance(scan, np.ndarray):
            scan = _f32(scan)
            st = lib.lsd_lio_scan(self.h, _ptr(scan), scan.shape[0], _ptr(state), _ptr(P), C.byref(info))
        elif scan.is_cuda:
            st = lib.lsd_lio_scan_dev(self.h, _ptr(scan), scan.shape[0], _ptr(state), _ptr(P), C.byref(info))
        else:  # pinned / pageable host torch tensor
            st = lib.lsd_lio_scan(self.h, _ptr(scan), scan.shape[0], _ptr(state), _ptr(P), C.byref(info))
        check(st)
        self.n_down = info.n_down
        return state, P, dict(info.as_dict(), status=st)
