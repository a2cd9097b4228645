"""ctypes binding of the C ABI in include/srlivo_b200.h (libsrlivo_b200.so).

There is no CPU fallback: if the CUDA library is missing this module raises at load time, and every
compute entry point returns SRL_CUDA_ERROR when no GPU is present.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libsrlivo_b200.so")

SRL_OK, SRL_TOO_FEW_RESIDUALS, SRL_NAN_PLANARITY, SRL_CUDA_ERROR, SRL_BAD_ARG, SRL_MAP_FULL, SRL_SINGULAR, SRL_COMM_ERROR = range(8)
STATUS_NAMES = ["SRL_OK", "SRL_TOO_FEW_RESIDUALS", "SRL_NAN_PLANARITY", "SRL_CUDA_ERROR", "SRL_BAD_ARG", "SRL_MAP_FULL",
                "SRL_SINGULAR", "SRL_COMM_ERROR"]
NS = 17


class IcpParams(C.Structure):
    """srl_icp_params == the icpOptions fields read by the path (include/parameters.h:8-56)."""
    _fields_ = [
        ("size_voxel_map", C.c_double), ("power_planarity", C.c_double), ("max_dist_to_plane_icp", C.c_double),
        ("weight_alpha", C.c_double), ("weight_neighborhood", C.c_double), ("threshold_orientation_norm", C.c_double),
        ("threshold_translation_norm", C.c_double), ("laser_point_cov", C.c_double),
        ("voxel_neighborhood", C.c_int32), ("min_number_neighbors", C.c_int32), ("max_number_neighbors", C.c_int32),
        ("threshold_voxel_occupancy", C.c_int32), ("max_num_residuals", C.c_int32), ("num_iters_icp", C.c_int32),
        ("init_num_frames", C.c_int32), ("frame_id", C.c_int32),
    ]


class EskfState(C.Structure):
    _fields_ = [("p", C.c_double * 3), ("q", C.c_double * 4), ("v", C.c_double * 3), ("ba", C.c_double * 3),
                ("bg", C.c_double * 3), ("g", C.c_double * 3), ("cov", C.c_double * (NS * NS))]


class Frame(C.Structure):
    _fields_ = [("q_cur", C.c_double * 4), ("t_cur", C.c_double * 3), ("t_last", C.c_double * 3),
                ("R_il", C.c_double * 9), ("t_il", C.c_double * 3)]


class NormalEq(C.Structure):
    _fields_ = [("HTH", C.c_double * 36), ("HTh", C.c_double * 6), ("loss_sum", C.c_double),
                ("num_residuals", C.c_int64), ("num_full_neighborhoods", C.c_int64),
                ("num_candidates_scanned", C.c_int64), ("num_keypoints", C.c_int64),
                ("nan_planarity", C.c_int32), ("reserved", C.c_int32)]


class DebugOut(C.Structure):
    _fields_ = [("world_xyz", C.c_void_p), ("status", C.c_void_p), ("nbr", C.c_void_p), ("nbr_dist", C.c_void_p),
                ("plane", C.c_void_p)]


class IekfSummary(C.Structure):
    _fields_ = [("success", C.c_int32), ("passes_run", C.c_int32), ("num_residuals_used", C.c_int32),
                ("converged", C.c_int32), ("trace", (C.c_double * 24) * 32)]


class ImuState(C.Structure):
    """srl_imu_state: the imuState fields the point transforms read (include/utility.h)."""
    _fields_ = [("timestamp", C.c_double), ("quat", C.c_double * 4), ("trans", C.c_double * 3), ("vel", C.c_double * 3),
                ("un_acc", C.c_double * 3), ("un_gyr", C.c_double * 3)]


class Camera(C.Structure):
    """srl_camera: the state fields cloudFrame::project3dTo2d / if2dPointsAvailable read (include/state.h)."""
    _fields_ = [("q_camera_world", C.c_double * 4), ("t_camera_world", C.c_double * 3), ("t_world_camera", C.c_double * 3),
                ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double), ("fov_margin", C.c_double),
                ("cols", C.c_int32), ("rows", C.c_int32)]


class LkParams(C.Structure):
    """srl_lk_params: LKOpticalFlowKernel's constructor arguments (include/lkpyramid.h:100-106)."""
    _fields_ = [("win_w", C.c_int32), ("win_h", C.c_int32), ("max_level", C.c_int32), ("criteria_type", C.c_int32), ("max_count", C.c_int32),
                ("epsilon", C.c_double), ("flags", C.c_int32), ("min_eig_threshold", C.c_double)]


class ImageParams(C.Structure):
    """srl_image_params: the yaml's camera_parameter values imageProcessing is given (src/imageProcessing.cpp:32-53)."""
    _fields_ = [("image_width", C.c_int32), ("image_height", C.c_int32), ("camera_intrinsic", C.c_double * 9),
                ("camera_dist_coeffs", C.c_double * 5)]


class VioState(C.Structure):
    """srl_vio_state: the p_state fields vioEsikf / vioPhotometric read and write (include/state.h); quaternions x, y, z, w."""
    _fields_ = [("rotation", C.c_double * 4), ("translation", C.c_double * 3), ("R_imu_camera", C.c_double * 9),
                ("t_imu_camera", C.c_double * 3), ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("time_td", C.c_double), ("q_world_camera", C.c_double * 4), ("t_world_camera", C.c_double * 3),
                ("q_camera_world", C.c_double * 4), ("t_camera_world", C.c_double * 3)]


class ProjectionParams(C.Structure):
    """srl_projection_params: the arguments of rgbMapTracker::selectPointsForProjection and the tracker's depth bounds."""
    _fields_ = [("minimum_dis", C.c_double), ("skip_step", C.c_int32), ("use_all_points", C.c_int32), ("minimum_depth", C.c_double),
                ("maximum_depth", C.c_double)]


class FlowTrackerSets(C.Structure):
    """srl_flow_tracker_sets_out: the optical-flow tracker's set counts and device pointers."""
    _fields_ = [("n_match", C.c_int64), ("n_cur", C.c_int64), ("n_last", C.c_int64), ("match_ids", C.c_void_p),
                ("match_last_uv", C.c_void_p), ("match_uv", C.c_void_p), ("cur_ids", C.c_void_p), ("cur_uv", C.c_void_p),
                ("cur_velocity", C.c_void_p), ("last_ids", C.c_void_p), ("last_uv", C.c_void_p), ("last_image_time", C.c_double)]


class BuildFrameParams(C.Structure):
    """srl_build_frame_params: buildFrame's inputs (src/lioOptimization.cpp:821-893)."""
    _fields_ = [("timestamp_begin", C.c_double), ("timestamp_offset", C.c_double), ("point_time_enable", C.c_int32),
                ("motion_compensation", C.c_int32), ("index_frame", C.c_int32), ("init_num_frames", C.c_int32),
                ("init_voxel_size", C.c_double), ("voxel_size", C.c_double), ("R_il", C.c_double * 9), ("t_il", C.c_double * 3),
                ("q_pred", C.c_double * 4), ("t_pred", C.c_double * 3), ("prev_time_sweep_end", C.c_double)]


class BuildFrameInfo(C.Structure):
    """srl_build_frame_info: the cloudFrame scalars and what each stage did."""
    _fields_ = [("time_sweep_begin", C.c_double), ("time_sweep_end", C.c_double), ("time_frame_begin", C.c_double),
                ("time_frame_end", C.c_double), ("offset_begin", C.c_double), ("offset_end", C.c_double), ("dt_offset", C.c_double),
                ("sample_size", C.c_double), ("frame_id", C.c_int32), ("reserved", C.c_int32), ("n_input", C.c_int64),
                ("n_timestamped", C.c_int64), ("n_imu_written", C.c_int64), ("n_points", C.c_int64), ("engine_words", C.c_int64),
                ("shuffle_rejections", C.c_int64), ("stage_ms", C.c_double * 6)]


class CloudFramePtrs(C.Structure):
    _fields_ = [("raw_point", C.c_void_p), ("point", C.c_void_p), ("imu_point", C.c_void_p), ("relative_time", C.c_void_p),
                ("alpha_time", C.c_void_p), ("timestamp", C.c_void_p), ("source_index", C.c_void_p)]


class LidarParams(C.Structure):
    """srl_lidar_params: cloudProcessing's configuration (lidar_parameter / common in the reference's yaml)."""
    _fields_ = [("lidar_type", C.c_int32), ("n_scans", C.c_int32), ("scan_rate", C.c_int32), ("time_unit", C.c_int32),
                ("blind", C.c_double), ("point_filter_num", C.c_int32), ("reserved", C.c_int32)]


class Cloud2Layout(C.Structure):
    _fields_ = [("point_step", C.c_uint32), ("off_x", C.c_int32), ("off_y", C.c_int32), ("off_z", C.c_int32),
                ("off_time", C.c_int32), ("off_ring", C.c_int32), ("width", C.c_uint32), ("row_step", C.c_uint32)]


class LidarInfo(C.Structure):
    _fields_ = [("last_end_time", C.c_double), ("given_offset_time", C.c_int32), ("sweep_id", C.c_int32),
                ("sweep_interval", C.c_double), ("size", C.c_int64), ("front_timestamp", C.c_double),
                ("back_timestamp", C.c_double), ("capacity", C.c_int64)]


class IekfIter(C.Structure):
    _fields_ = [("predict", EskfState), ("pass_index", C.c_int32), ("max_num_iter", C.c_int32)]


# every symbol include/srlivo_b200.h declares (tests check the library exports all of them)
EXPORTS = [
    "srl_abi_version", "srl_build_info", "srl_icp_params_r3live", "srl_ctx_create", "srl_ctx_destroy",
    "srl_last_error", "srl_ctx_synchronize", "srl_ctx_kernel_launches", "srl_ctx_set_timing", "srl_ctx_pass_time", "srl_ctx_set_option", "srl_ctx_get_counter", "srl_map_create", "srl_map_destroy",
    "srl_map_clear", "srl_map_stats", "srl_map_remove_far", "srl_map_upload", "srl_map_download", "srl_map_insert",
    "srl_map_insert_device", "srl_map_insert_sweep", "srl_sweep_create", "srl_sweep_destroy", "srl_sweep_upload", "srl_sweep_set_device",
    "srl_sweep_set_shard", "srl_sweep_download_order", "srl_build_plane_residuals", "srl_build_plane_residuals_async", "srl_normal_eq_unpack",
    "srl_iekf_begin", "srl_iekf_step", "srl_update_iekf", "srl_comm_create", "srl_comm_destroy", "srl_comm_export", "srl_comm_connect",
    "srl_update_iekf_dist", "srl_optimize_host", "srl_optimize_host_dist", "srl_shard_range", "srl_sweep_transform_device",
    "srl_grid_sampling", "srl_eskf_observe", "srl_host_plane_fit", "srl_iekf_replay",
    "srl_distort_frame_by_constant", "srl_distort_frame_by_imu", "srl_transform_all_imu_point",
    "srl_color_map_create", "srl_color_map_destroy", "srl_color_map_voxels", "srl_color_map_stats", "srl_color_map_add_points",
    "srl_color_map_render_recent", "srl_color_map_download_state", "srl_color_map_download_lists",
    "srl_map_create_growable", "srl_map_capacity", "srl_color_map_create_growable", "srl_color_map_capacity",
    "srl_cloud_frame_create", "srl_cloud_frame_destroy", "srl_cloud_frame_size", "srl_cloud_frame_device", "srl_cloud_frame_download",
    "srl_build_frame", "srl_shuffle_replay", "srl_map_insert_published", "srl_map_insert_sweep_published", "srl_color_map_export",
    "srl_color_map_select_for_projection", "srl_color_map_gather_points",
    "srl_lk_create", "srl_lk_destroy", "srl_lk_track_image", "srl_lk_info", "srl_lk_download_level", "srl_lk_last_times",
    "srl_image_create", "srl_image_destroy", "srl_image_process", "srl_image_info", "srl_image_download_maps", "srl_image_last_times",
    "srl_image_vio_esikf", "srl_image_vio_photometric", "srl_image_covariance", "srl_image_vio_last_summary", "srl_image_vio_last_times",
    "srl_flow_tracker_create", "srl_flow_tracker_destroy", "srl_flow_tracker_init", "srl_flow_tracker_track_image",
    "srl_flow_tracker_reject_matches", "srl_flow_tracker_remove_outliers", "srl_flow_tracker_update_and_append", "srl_flow_tracker_sets",
    "srl_flow_tracker_outlier_counts",
    "srl_lidar_create", "srl_lidar_destroy", "srl_lidar_livox", "srl_lidar_process", "srl_lidar_cut", "srl_lidar_info_get",
    "srl_lidar_download", "srl_lidar_sort_replay",
]

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback for the scan-matching path)")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, dbl, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_double, C.c_size_t
    L.srl_abi_version.restype = C.c_int
    L.srl_build_info.restype = C.c_char_p
    L.srl_icp_params_r3live.argtypes = [C.POINTER(IcpParams)]
    L.srl_ctx_create.argtypes = [C.c_int, vp, C.POINTER(vp)]
    L.srl_ctx_destroy.argtypes = [vp]
    L.srl_ctx_destroy.restype = None
    L.srl_last_error.argtypes = [vp]
    L.srl_last_error.restype = C.c_char_p
    L.srl_ctx_synchronize.argtypes = [vp]
    L.srl_ctx_kernel_launches.argtypes = [vp]
    L.srl_ctx_kernel_launches.restype = i64
    L.srl_ctx_set_option.argtypes = [vp, C.c_char_p, i64]
    L.srl_ctx_get_counter.argtypes = [vp, C.c_char_p, C.POINTER(i64)]
    L.srl_ctx_set_timing.argtypes = [vp, C.c_int]
    L.srl_ctx_pass_time.argtypes = [vp, C.POINTER(dbl), C.POINTER(i64), C.c_int]
    L.srl_map_create.argtypes = [vp, dbl, i32, sz, C.POINTER(vp)]
    L.srl_map_create_growable.argtypes = [vp, dbl, i32, sz, sz, C.POINTER(vp)]
    L.srl_map_capacity.argtypes = [vp] + [C.POINTER(sz)] * 3
    L.srl_map_destroy.argtypes = [vp]
    L.srl_map_destroy.restype = None
    L.srl_map_clear.argtypes = [vp]
    L.srl_map_stats.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
    L.srl_map_remove_far.argtypes = [vp, vp, dbl, C.POINTER(i64)]
    L.srl_map_upload.argtypes = [vp, vp, vp, vp, sz]
    L.srl_map_download.argtypes = [vp, vp, vp, vp, sz, C.POINTER(i64)]
    L.srl_map_insert.argtypes = [vp, vp, sz, dbl, i32, C.POINTER(i64)]
    L.srl_map_insert_device.argtypes = [vp, vp, sz, dbl, i32, C.POINTER(i64)]
    L.srl_map_insert_sweep.argtypes = [vp, vp, vp, vp, vp, vp, dbl, i32, C.POINTER(i64)]
    L.srl_map_insert_published.argtypes = [vp, vp, sz, dbl, i32, dbl, vp, sz, C.POINTER(i64), C.POINTER(i64)]
    L.srl_map_insert_sweep_published.argtypes = [vp, vp, vp, vp, vp, vp, dbl, i32, vp, sz, C.POINTER(i64), C.POINTER(i64)]
    L.srl_sweep_create.argtypes = [vp, sz, C.POINTER(vp)]
    L.srl_sweep_destroy.argtypes = [vp]
    L.srl_sweep_destroy.restype = None
    L.srl_sweep_upload.argtypes = [vp, vp, sz]
    L.srl_sweep_set_device.argtypes = [vp, vp, sz]
    L.srl_sweep_set_shard.argtypes = [vp, sz, sz]
    L.srl_sweep_download_order.argtypes = [vp, vp, sz, C.POINTER(i64)]
    L.srl_build_plane_residuals.argtypes = [vp, vp, vp, C.POINTER(Frame), C.POINTER(IcpParams), C.POINTER(NormalEq),
                                            C.POINTER(DebugOut)]
    L.srl_build_plane_residuals_async.argtypes = [vp, vp, vp, C.POINTER(Frame), C.POINTER(IcpParams), vp]
    L.srl_normal_eq_unpack.argtypes = [vp, C.POINTER(NormalEq)]
    L.srl_iekf_begin.argtypes = [C.POINTER(EskfState), C.POINTER(IcpParams), C.POINTER(IekfIter)]
    L.srl_iekf_step.argtypes = [C.POINTER(IekfIter), C.POINTER(NormalEq), C.POINTER(IcpParams), C.POINTER(EskfState),
                                vp, vp, vp, C.POINTER(i32), C.POINTER(i32)]
    L.srl_update_iekf.argtypes = [vp, vp, vp, C.POINTER(EskfState), vp, vp, vp, vp, vp, C.POINTER(IcpParams),
                                  C.POINTER(IekfSummary)]
    L.srl_comm_create.argtypes = [vp, C.c_int, C.c_int, C.POINTER(vp)]
    L.srl_comm_destroy.argtypes = [vp]
    L.srl_comm_destroy.restype = None
    L.srl_comm_export.argtypes = [vp, vp]
    L.srl_comm_connect.argtypes = [vp, vp]
    L.srl_update_iekf_dist.argtypes = [vp, vp, vp, vp, C.POINTER(EskfState), vp, vp, vp, vp, vp, C.POINTER(IcpParams),
                                       C.POINTER(IekfSummary)]
    L.srl_optimize_host.argtypes = [vp, vp, vp, vp, sz, C.POINTER(EskfState), vp, vp, vp, vp, vp, C.POINTER(IcpParams),
                                    C.POINTER(IekfSummary), vp]
    L.srl_optimize_host_dist.argtypes = [vp, vp, vp, vp, vp, sz, C.POINTER(EskfState), vp, vp, vp, vp, vp, C.POINTER(IcpParams),
                                         C.POINTER(IekfSummary), vp, C.POINTER(sz), C.POINTER(sz)]
    L.srl_shard_range.argtypes = [sz, C.c_int, C.c_int, C.POINTER(sz), C.POINTER(sz)]
    L.srl_shard_range.restype = None
    L.srl_sweep_transform_device.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.srl_grid_sampling.argtypes = [vp, vp, sz, dbl, vp, C.POINTER(sz)]
    L.srl_eskf_observe.argtypes = [C.POINTER(EskfState), vp]
    L.srl_distort_frame_by_constant.argtypes = [vp, vp, vp, sz, vp, sz, dbl, vp, vp, vp]
    L.srl_distort_frame_by_imu.argtypes = [vp, vp, vp, sz, vp, sz, dbl, vp, vp, vp, C.POINTER(i64)]
    L.srl_transform_all_imu_point.argtypes = [vp, vp, sz, vp, vp, vp, vp]
    L.srl_host_plane_fit.argtypes = [vp, i32, vp, vp, vp]
    L.srl_iekf_replay.argtypes = [vp, C.POINTER(EskfState), vp, vp, C.POINTER(IcpParams), vp, i32, i64, C.POINTER(IekfSummary)]
    L.srl_color_map_create.argtypes = [vp, dbl, i32, sz, dbl, C.POINTER(vp)]
    L.srl_color_map_create_growable.argtypes = [vp, dbl, i32, sz, sz, dbl, C.POINTER(vp)]
    L.srl_color_map_capacity.argtypes = [vp] + [C.POINTER(sz)] * 4
    L.srl_color_map_destroy.argtypes = [vp]
    L.srl_color_map_destroy.restype = None
    L.srl_color_map_voxels.argtypes = [vp]
    L.srl_color_map_voxels.restype = vp
    L.srl_color_map_stats.argtypes = [vp] + [C.POINTER(i64)] * 5
    L.srl_color_map_add_points.argtypes = [vp, vp, sz, i32, dbl, dbl, i32, C.POINTER(i64)]
    L.srl_color_map_render_recent.argtypes = [vp, C.POINTER(Camera), vp, dbl, C.POINTER(i64)]
    L.srl_color_map_download_state.argtypes = [vp, sz, vp, vp, vp, vp, vp, vp]
    L.srl_color_map_download_lists.argtypes = [vp, vp, vp]
    L.srl_color_map_export.argtypes = [vp, i32, i32, vp, vp, sz, C.POINTER(i64)]
    L.srl_color_map_select_for_projection.argtypes = [vp, C.POINTER(Camera), C.POINTER(ProjectionParams), vp, vp, vp, sz, C.POINTER(i64)]
    L.srl_color_map_gather_points.argtypes = [vp, vp, sz, vp, vp, vp, vp, vp]
    L.srl_lk_create.argtypes = [vp, C.POINTER(LkParams), C.POINTER(vp)]
    L.srl_lk_destroy.argtypes = [vp]
    L.srl_lk_destroy.restype = None
    L.srl_lk_track_image.argtypes = [vp, vp, C.c_int, C.c_int, sz, vp, sz, vp, vp, C.POINTER(i64)]
    L.srl_lk_info.argtypes = [vp] + [C.POINTER(i32)] * 3
    L.srl_lk_download_level.argtypes = [vp, C.c_int, C.c_int, vp, vp]
    L.srl_lk_last_times.argtypes = [vp, C.POINTER(dbl), C.POINTER(dbl)]
    L.srl_image_create.argtypes = [vp, C.POINTER(ImageParams), C.c_int, C.c_int, C.POINTER(vp)]
    L.srl_image_destroy.argtypes = [vp]
    L.srl_image_destroy.restype = None
    L.srl_image_process.argtypes = [vp, vp, C.c_int, C.c_int, sz, vp, vp]
    L.srl_image_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(dbl), vp]
    L.srl_image_download_maps.argtypes = [vp, vp, vp]
    L.srl_image_last_times.argtypes = [vp, C.POINTER(dbl), C.POINTER(dbl), C.POINTER(dbl)]
    L.srl_image_vio_esikf.argtypes = [vp, vp, C.POINTER(VioState), vp, vp, vp, sz, i32, C.POINTER(i32)]
    L.srl_image_vio_photometric.argtypes = [vp, vp, C.POINTER(VioState), vp, vp, sz, i32, vp, C.c_int, C.c_int, sz, C.POINTER(i32)]
    L.srl_image_covariance.argtypes = [vp, vp, vp]
    L.srl_image_vio_last_summary.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(dbl)]
    L.srl_image_vio_last_times.argtypes = [vp, C.POINTER(dbl), C.POINTER(dbl)]
    L.srl_flow_tracker_create.argtypes = [vp, vp, vp, i32, C.POINTER(vp)]
    L.srl_flow_tracker_destroy.argtypes = [vp]
    L.srl_flow_tracker_destroy.restype = None
    L.srl_flow_tracker_init.argtypes = [vp, vp, C.c_int, C.c_int, sz, dbl, vp, vp, sz]
    L.srl_flow_tracker_track_image.argtypes = [vp, vp, C.c_int, C.c_int, sz, dbl, C.POINTER(i32)]
    L.srl_flow_tracker_reject_matches.argtypes = [vp, vp, sz]
    L.srl_flow_tracker_remove_outliers.argtypes = [vp, vp, sz, C.POINTER(i32)]
    L.srl_flow_tracker_update_and_append.argtypes = [vp, C.POINTER(Camera), dbl, vp, sz]
    L.srl_flow_tracker_sets.argtypes = [vp, C.POINTER(FlowTrackerSets)]
    L.srl_flow_tracker_outlier_counts.argtypes = [vp, vp, sz, vp]
    L.srl_lidar_create.argtypes = [vp, C.POINTER(LidarParams), sz, C.POINTER(vp)]
    L.srl_lidar_destroy.argtypes = [vp]
    L.srl_lidar_destroy.restype = None
    L.srl_lidar_livox.argtypes = [vp, vp, sz, sz, dbl, C.POINTER(i64)]
    L.srl_lidar_process.argtypes = [vp, vp, sz, C.POINTER(Cloud2Layout), dbl, C.POINTER(i64)]
    L.srl_lidar_cut.argtypes = [vp, dbl, C.POINTER(i64), C.POINTER(vp), C.POINTER(vp)]
    L.srl_lidar_info_get.argtypes = [vp, C.POINTER(LidarInfo)]
    L.srl_lidar_download.argtypes = [vp, vp, vp, vp]
    L.srl_lidar_sort_replay.argtypes = [vp, vp, sz, vp, C.POINTER(i32)]
    L.srl_cloud_frame_create.argtypes = [vp, sz, C.POINTER(vp)]
    L.srl_cloud_frame_destroy.argtypes = [vp]
    L.srl_cloud_frame_destroy.restype = None
    L.srl_cloud_frame_size.argtypes = [vp]
    L.srl_cloud_frame_size.restype = sz
    L.srl_cloud_frame_device.argtypes = [vp, C.POINTER(CloudFramePtrs)]
    L.srl_cloud_frame_download.argtypes = [vp] + [vp] * 7
    L.srl_build_frame.argtypes = [vp, vp, vp, sz, vp, sz, C.POINTER(BuildFrameParams), vp, C.POINTER(BuildFrameInfo)]
    L.srl_shuffle_replay.argtypes = [vp, vp, sz, sz, i32, vp, C.POINTER(sz), C.POINTER(C.c_uint64)]
    _lib = L
    return L


class SrlError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"{STATUS_NAMES[code] if 0 <= code < len(STATUS_NAMES) else code}: {msg}")
        self.code = code


def r3live_params(**kw) -> IcpParams:
    p = IcpParams()
    lib().srl_icp_params_r3live(C.byref(p))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def eskf_to_c(p, q, v, ba, bg, g, cov) -> EskfState:
    """One memmove of the 308 doubles (p3 q4 v3 ba3 bg3 g3 cov289) instead of per-element ctypes stores (~50 us)."""
    packed = np.empty(19 + NS * NS, np.float64)
    packed[0:3] = p; packed[3:7] = q; packed[7:10] = v; packed[10:13] = ba; packed[13:16] = bg; packed[16:19] = g
    packed[19:] = np.asarray(cov, np.float64).reshape(-1)
    s = EskfState()
    C.memmove(C.addressof(s), packed.ctypes.data, packed.nbytes)
    return s


def eskf_from_c(s: EskfState) -> dict:
    a = np.frombuffer(s, dtype=np.float64, count=19 + NS * NS).copy()
    return dict(p=a[0:3], q=a[3:7], v=a[7:10], ba=a[10:13], bg=a[13:16], g=a[16:19], cov=a[19:].reshape(NS, NS))


def summary_trace(summ: "IekfSummary") -> np.ndarray:
    """The per-pass trace rows of an srl_iekf_summary as a (passes, 24) array."""
    n = min(int(summ.passes_run), 32)
    return np.frombuffer(summ, dtype=np.float64, count=32 * 24, offset=IekfSummary.trace.offset).reshape(32, 24)[:n].copy()
