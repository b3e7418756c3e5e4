"""ctypes binding of libkicp_b200.so (include/kicp.h).  There is no CPU fallback: if the shared library is missing
the import fails loudly, and without a CUDA device every call raises KicpError."""
import ctypes as C
import os

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.normpath(os.path.join(_PKG, "..", ".."))  # kinematic-icp_b200/
LIB_PATH = os.environ.get("KICP_LIB", os.path.join(_ROOT, "lib", "libkicp_b200.so"))  # KICP_LIB: A/B builds of the same ABI
KICP_MAX_ITERATIONS = 64
KICP_UNIQUE_ID_BYTES = 128
KICP_IPC_HANDLE_BYTES = 64

KICP_OK = 0
KICP_ERR_CUDA, KICP_ERR_INVALID, KICP_ERR_UNSUPPORTED, KICP_ERR_NCCL, KICP_ERR_CAPACITY = 1, 2, 3, 4, 5
KICP_WARN_NO_CORRESPONDENCES = 16

c_dp = C.POINTER(C.c_double)
c_fp = C.POINTER(C.c_float)
c_ip = C.POINTER(C.c_int32)


class RegParams(C.Structure):
    """kicp_reg_params — the public fields of kinematic_icp::KinematicRegistration (Registration.hpp:45-49)."""
    _fields_ = [("max_num_iterations", C.c_int32), ("use_adaptive_odometry_regularization", C.c_int32),
                ("convergence_criterion", C.c_double), ("fixed_regularization", C.c_double)]


class RegResult(C.Structure):
    """kicp_reg_result"""
    _fields_ = [("pose", C.c_double * 7), ("beta", C.c_double), ("last_dx_norm", C.c_double), ("iterations", C.c_int32),
                ("status", C.c_int32), ("sums", (C.c_double * 8) * KICP_MAX_ITERATIONS),
                ("dx", (C.c_double * 2) * KICP_MAX_ITERATIONS)]

    def pose_np(self):
        return np.array(self.pose[:], dtype=np.float64)

    def sums_np(self):
        return np.ctypeslib.as_array(self.sums)[: self.iterations].copy()

    def dx_np(self):
        return np.ctypeslib.as_array(self.dx)[: self.iterations].copy()


class Profile(C.Structure):
    """kicp_profile"""
    _fields_ = [("assoc_ms", C.c_double), ("assoc_launches", C.c_int64), ("idle_ms", C.c_double),
                ("idle_launches", C.c_int64), ("prep_ms", C.c_double), ("registrations", C.c_int64),
                ("assoc_iterations", C.c_int64)]


class CorrStats(C.Structure):
    """kicp_corr_stats: a cloud's correspondences at a pose (kicp_map_correspondences, option "correspondences" of the frame calls)"""
    _fields_ = [("n_points", C.c_int64), ("n_inliers", C.c_int64), ("fitness", C.c_double), ("inlier_rmse", C.c_double),
                ("sum_sq", C.c_double), ("jtj", C.c_double * 3), ("jtr", C.c_double * 2)]


class PoseSearchParams(C.Structure):
    """kicp_pose_search_params"""
    _fields_ = [("half_extent", C.c_double * 3), ("step", C.c_double * 3), ("tau", C.c_double), ("levels", C.c_int32), ("keep", C.c_int32)]


class PoseHypothesis(C.Structure):
    """kicp_pose_hypothesis"""
    _fields_ = [("pose", C.c_double * 7), ("offset", C.c_double * 3), ("lattice", C.c_int32 * 3), ("level", C.c_int32),
                ("n_inliers", C.c_int64), ("fitness", C.c_double), ("inlier_rmse", C.c_double), ("sum_sq", C.c_double)]


KICP_ALIGN_CONVERGED, KICP_ALIGN_MAX_ITERATIONS, KICP_ALIGN_NO_CORRESPONDENCES, KICP_ALIGN_SINGULAR = 0, 1, 2, 3


class PlanarAlignParams(C.Structure):
    """kicp_planar_align_params"""
    _fields_ = [("tau", C.c_double), ("convergence", C.c_double), ("max_iterations", C.c_int32)]


class PlanarAlignment(C.Structure):
    """kicp_planar_alignment"""
    _fields_ = [("pose", C.c_double * 7), ("status", C.c_int32), ("iterations", C.c_int32), ("last_step", C.c_double),
                ("n_inliers", C.c_int64), ("fitness", C.c_double), ("inlier_rmse", C.c_double), ("sum_sq", C.c_double),
                ("jtj", C.c_double * 6), ("jtr", C.c_double * 3)]


KICP_MAP_UPDATE_ALWAYS, KICP_MAP_UPDATE_NEVER, KICP_MAP_UPDATE_GATED = 0, 1, 2
KICP_FRAME_UPDATE_APPLIED, KICP_FRAME_UPDATE_NO_CORRESPONDENCES, KICP_FRAME_UPDATE_REJECTED, KICP_FRAME_UPDATE_SKIPPED, \
    KICP_FRAME_UPDATE_NONE = 0, 1, 2, 3, 4


class MapUpdatePolicy(C.Structure):
    """kicp_map_update_policy"""
    _fields_ = [("mode", C.c_int32), ("min_inliers", C.c_int64), ("min_fitness", C.c_double), ("max_inlier_rmse", C.c_double)]


class FreeSpaceParams(C.Structure):
    """kicp_free_space_params"""
    _fields_ = [("end_margin", C.c_double), ("min_misses", C.c_int32)]


class FreeSpaceStats(C.Structure):
    """kicp_free_space_stats"""
    _fields_ = [("rays", C.c_int64), ("visits", C.c_int64), ("cleared_voxels", C.c_int64), ("cleared_points", C.c_int64),
                ("prior_contradicted", C.c_int64)]


class OccupancyParams(C.Structure):
    """kicp_occupancy_params"""
    _fields_ = [("initial", C.c_int32), ("hit_gain", C.c_int32), ("miss_loss", C.c_int32), ("max_evidence", C.c_int32)]


class FrameInput(C.Structure):
    """kicp_frame_input"""
    _fields_ = [("data", C.c_void_p), ("n", C.c_int64), ("dtype", C.c_int32), ("point_step", C.c_int32), ("offset_x", C.c_int32),
                ("offset_y", C.c_int32), ("offset_z", C.c_int32), ("stamps", c_dp), ("n_stamps", C.c_int64)]


class FrameParams(C.Structure):
    """kicp_frame_params"""
    _fields_ = [("max_range", C.c_double), ("min_range", C.c_double), ("deskew", C.c_int32), ("voxel_size", C.c_double),
                ("stage_clouds", C.c_int32), ("reg", RegParams)]


class LaserScan(C.Structure):
    """kicp_laser_scan — sensor_msgs/msg/LaserScan without header and intensities"""
    _fields_ = [("ranges", c_fp), ("n", C.c_int64), ("angle_min", C.c_float), ("angle_max", C.c_float), ("angle_increment", C.c_float),
                ("time_increment", C.c_float), ("range_min", C.c_float), ("range_max", C.c_float)]


class SensorInput(C.Structure):
    """kicp_sensor_input"""
    _fields_ = [("kind", C.c_int32), ("device", C.c_int32), ("points", FrameInput), ("stamp_datatype", C.c_int32), ("stamp_offset", C.c_int32),
                ("scan", LaserScan), ("time_offset", C.c_double)]


class SensorStats(C.Structure):
    """kicp_sensor_stats"""
    _fields_ = [("n_points", C.c_int64), ("n_stamps", C.c_int64), ("stamp_range", C.c_double * 2)]


class MapLiveStats(C.Structure):
    """kicp_map_live_stats"""
    _fields_ = [("added", C.c_int64), ("removed", C.c_int64), ("moved", C.c_int64), ("rewritten", C.c_int64), ("written", C.c_int64)]


KICP_DTYPE_F64, KICP_DTYPE_F32 = 0, 1
KICP_MAP_LAYER_ALL, KICP_MAP_LAYER_PRIOR, KICP_MAP_LAYER_LIVE = 0, 1, 2  # kicp_map_pointcloud_layer
KICP_STAGE_F64, KICP_STAGE_F32 = 1, 2  # kicp_frame_params.stage_clouds flags
KICP_STAMP_NONE, KICP_STAMP_UINT32, KICP_STAMP_FLOAT32, KICP_STAMP_FLOAT64 = 0, 6, 7, 8  # PointField datatypes of a time field
KICP_MAX_SENSORS, KICP_SENSOR_POINTS, KICP_SENSOR_LASER_SCAN = 8, 0, 1
KICP_MAX_DESKEW_SEGMENTS = 64


class KicpError(RuntimeError):
    def __init__(self, status, where):
        self.status = status
        msg = lib().kicp_last_error().decode() if status in (KICP_ERR_CUDA, KICP_ERR_NCCL, KICP_ERR_CAPACITY,
                                                              KICP_ERR_UNSUPPORTED, KICP_ERR_INVALID) else ""
        super().__init__("%s: %s%s" % (where, lib().kicp_status_string(status).decode(), (" — " + msg) if msg else ""))


_LIB = None

# every symbol include/kicp.h declares: (name, restype, argtypes)
_P = C.c_void_p
SYMBOLS = [
    ("kicp_status_string", C.c_char_p, [C.c_int]),
    ("kicp_last_error", C.c_char_p, []),
    ("kicp_ctx_create", C.c_int, [C.c_int, C.POINTER(_P)]),
    ("kicp_ctx_destroy", C.c_int, [_P]),
    ("kicp_ctx_synchronize", C.c_int, [_P]),
    ("kicp_ctx_stream", _P, [_P]),
    ("kicp_ctx_launch_count", C.c_int64, [_P]),
    ("kicp_ctx_wait_stream", C.c_int, [_P, _P]),
    ("kicp_stream_wait_ctx", C.c_int, [_P, _P]),
    ("kicp_ctx_set_option", C.c_int, [_P, C.c_char_p, C.c_int32]),
    ("kicp_ctx_profile_begin", C.c_int, [_P]),
    ("kicp_ctx_profile_end", C.c_int, [_P, C.POINTER(Profile)]),
    ("kicp_host_alloc", C.c_int, [C.c_uint64, C.POINTER(_P)]),
    ("kicp_host_free", C.c_int, [_P]),
    ("kicp_map_create", C.c_int, [_P, C.c_double, C.c_double, C.c_uint32, C.POINTER(_P)]),
    ("kicp_map_destroy", C.c_int, [_P]),
    ("kicp_map_reserve", C.c_int, [_P, C.c_int64]),
    ("kicp_map_clear", C.c_int, [_P]),
    ("kicp_map_empty", C.c_int, [_P, c_ip]),
    ("kicp_map_num_points", C.c_int, [_P, C.POINTER(C.c_int64)]),
    ("kicp_map_num_voxels", C.c_int, [_P, C.POINTER(C.c_int64)]),
    ("kicp_map_add_points", C.c_int, [_P, c_dp, C.c_int64]),
    ("kicp_map_remove_far", C.c_int, [_P, c_dp]),
    ("kicp_map_update", C.c_int, [_P, c_dp, C.c_int64, c_dp]),
    ("kicp_map_update_pose", C.c_int, [_P, c_dp, C.c_int64, c_dp]),
    ("kicp_map_pointcloud", C.c_int, [_P, c_dp, C.c_int64, C.POINTER(C.c_int64)]),
    ("kicp_map_pointcloud_f32", C.c_int, [_P, c_fp, C.c_int64, C.POINTER(C.c_int64)]),
    ("kicp_map_pointcloud_device_async", C.c_int, [_P, _P, C.c_int32, C.c_int64, C.POINTER(C.c_int64)]),
    ("kicp_map_pointcloud_f32_live", C.c_int, [_P, C.POINTER(c_fp), C.POINTER(C.c_int64), C.POINTER(MapLiveStats)]),
    ("kicp_map_export_voxels", C.c_int, [_P, c_ip, c_ip, c_dp, C.c_int64, C.c_int64, C.POINTER(C.c_int64),
                                         C.POINTER(C.c_int64)]),
    ("kicp_map_load_voxels", C.c_int, [_P, c_ip, c_ip, c_dp, C.c_int64]),
    ("kicp_map_freeze", C.c_int, [_P]),
    ("kicp_map_thaw", C.c_int, [_P]),
    ("kicp_map_prior_size", C.c_int, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    ("kicp_map_pointcloud_layer", C.c_int, [_P, C.c_int32, C.c_int32, _P, C.c_int64, C.POINTER(C.c_int64)]),
    ("kicp_map_pointcloud_layer_device_async", C.c_int, [_P, C.c_int32, C.c_int32, _P, C.c_int64, C.POINTER(C.c_int64)]),
    ("kicp_map_clear_free_space", C.c_int, [_P, c_dp, C.c_int64, c_dp, c_dp, C.POINTER(FreeSpaceParams), C.POINTER(FreeSpaceStats)]),
    ("kicp_map_clear_free_space_device", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, c_dp, c_dp,
                                                   C.POINTER(FreeSpaceParams), C.POINTER(FreeSpaceStats)]),
    ("kicp_map_set_occupancy", C.c_int, [_P, C.POINTER(OccupancyParams)]),
    ("kicp_map_export_occupancy", C.c_int, [_P, c_ip, C.c_int64, C.POINTER(C.c_int64)]),
    ("kicp_map_nearest", C.c_int, [_P, c_dp, C.c_int64, c_dp, c_dp]),
    ("kicp_map_add_points_device", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    ("kicp_map_update_device", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, c_dp]),
    ("kicp_map_update_pose_device", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, c_dp]),
    ("kicp_map_nearest_device_async", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    ("kicp_map_correspondences", C.c_int, [_P, c_dp, C.c_int64, c_dp, C.c_double, c_dp, c_dp, _P, C.POINTER(CorrStats)]),
    ("kicp_map_correspondences_device_async", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, c_dp,
                                                        C.c_double, _P, _P, _P, _P]),
    ("kicp_map_pose_search", C.c_int, [_P, c_dp, C.c_int64, c_dp, C.POINTER(PoseSearchParams), C.POINTER(PoseHypothesis), C.c_int32,
                                       C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    ("kicp_map_pose_search_device", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, c_dp,
                                              C.POINTER(PoseSearchParams), C.POINTER(PoseHypothesis), C.c_int32, C.POINTER(C.c_int32),
                                              C.POINTER(C.c_int64)]),
    ("kicp_map_align_planar", C.c_int, [_P, c_dp, C.c_int64, c_dp, C.c_int32, C.POINTER(PlanarAlignParams), C.POINTER(PlanarAlignment)]),
    ("kicp_map_align_planar_device", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, c_dp, C.c_int32,
                                               C.POINTER(PlanarAlignParams), C.POINTER(PlanarAlignment)]),
    ("kicp_voxel_downsample_device", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, _P, C.c_int64, C.POINTER(C.c_int64)]),
    ("kicp_preprocess_device", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, C.c_int64, c_dp, c_dp, C.c_double, C.c_double, C.c_int32, _P,
                                         C.c_int64, C.POINTER(C.c_int64)]),
    ("kicp_register", C.c_int, [_P, c_dp, C.c_int64, c_dp, c_dp, C.c_double, C.POINTER(RegParams), c_dp,
                                C.POINTER(RegResult)]),
    ("kicp_scan_create", C.c_int, [_P, C.c_int64, C.POINTER(_P)]),
    ("kicp_scan_destroy", C.c_int, [_P]),
    ("kicp_scan_upload", C.c_int, [_P, c_dp, C.c_int64]),
    ("kicp_scan_upload_async", C.c_int, [_P, c_dp, C.c_int64]),
    ("kicp_scan_upload_points", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    ("kicp_scan_upload_points_async", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    ("kicp_register_points", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, c_dp, c_dp,
                                       C.c_double, C.POINTER(RegParams), c_dp, C.POINTER(RegResult)]),
    ("kicp_register_scan_async", C.c_int, [_P, _P, c_dp, c_dp, C.c_double, C.POINTER(RegParams), C.POINTER(RegResult)]),
    ("kicp_scan_attach_device", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    ("kicp_voxel_downsample", C.c_int, [_P, c_dp, C.c_int64, C.c_double, c_dp, C.c_int64, C.POINTER(C.c_int64)]),
    ("kicp_preprocess", C.c_int, [_P, c_dp, C.c_int64, c_dp, C.c_int64, c_dp, c_dp, C.c_double, C.c_double, C.c_int32, c_dp,
                                  C.c_int64, C.POINTER(C.c_int64)]),
    ("kicp_register_frame", C.c_int, [_P, C.POINTER(FrameInput), c_dp, c_dp, c_dp, c_dp, C.c_double, C.POINTER(FrameParams), c_dp,
                                      c_dp, C.c_int64, C.POINTER(C.c_int64), c_dp, C.c_int64, C.POINTER(C.c_int64),
                                      C.POINTER(RegResult)]),
    ("kicp_frame_clouds", C.c_int, [_P, C.POINTER(c_dp), C.POINTER(C.c_int64), C.POINTER(c_dp), C.POINTER(C.c_int64)]),
    ("kicp_frame_clouds_f32", C.c_int, [_P, C.POINTER(c_fp), C.POINTER(C.c_int64), C.POINTER(c_fp), C.POINTER(C.c_int64)]),
    ("kicp_frame_clouds_device", C.c_int, [_P, C.c_int32, C.POINTER(_P), C.POINTER(C.c_int64), C.POINTER(_P), C.POINTER(C.c_int64)]),
    ("kicp_frame_correspondences", C.c_int, [_P, C.POINTER(CorrStats)]),
    ("kicp_frame_correspondences_device", C.c_int, [_P, C.POINTER(_P), C.POINTER(_P), C.POINTER(_P), C.POINTER(C.c_int64)]),
    ("kicp_ctx_set_map_update", C.c_int, [_P, C.POINTER(MapUpdatePolicy)]),
    ("kicp_frame_map_update", C.c_int, [_P, C.POINTER(C.c_int32)]),
    ("kicp_ctx_set_free_space", C.c_int, [_P, C.POINTER(FreeSpaceParams)]),
    ("kicp_frame_free_space", C.c_int, [_P, C.POINTER(FreeSpaceStats)]),
    ("kicp_frame_stage", C.c_int, [_P, C.POINTER(FrameInput), C.c_int32, C.c_int32, c_dp, C.POINTER(C.c_int64)]),
    ("kicp_frame_stage_device", C.c_int, [_P, C.POINTER(FrameInput), C.c_int32, C.c_int32, c_dp, C.POINTER(C.c_int64)]),
    ("kicp_register_staged_frame", C.c_int, [_P, c_dp, c_dp, c_dp, c_dp, C.c_double, C.POINTER(FrameParams), c_dp, c_dp, C.c_int64,
                                             C.POINTER(C.c_int64), c_dp, C.c_int64, C.POINTER(C.c_int64), C.POINTER(RegResult)]),
    ("kicp_frame_stage_laser_scan", C.c_int, [_P, C.POINTER(LaserScan), c_dp, C.POINTER(C.c_int64)]),
    ("kicp_frame_stage_laser_scan_device", C.c_int, [_P, C.POINTER(LaserScan), c_dp, C.POINTER(C.c_int64)]),
    ("kicp_frame_stage_sensors", C.c_int, [_P, C.POINTER(SensorInput), C.c_int32, c_dp, C.POINTER(SensorStats)]),
    ("kicp_register_staged_sensors", C.c_int, [_P, C.c_int32, c_dp, c_dp, c_dp, c_dp, C.c_double, C.POINTER(FrameParams), c_dp, c_dp,
                                               C.c_int64, C.POINTER(C.c_int64), c_dp, C.c_int64, C.POINTER(C.c_int64), C.POINTER(RegResult)]),
    ("kicp_register_staged_frame_segments", C.c_int, [_P, C.c_int32, c_dp, c_dp, c_dp, c_dp, C.c_double, C.POINTER(FrameParams), c_dp,
                                                      c_dp, C.c_int64, C.POINTER(C.c_int64), c_dp, C.c_int64, C.POINTER(C.c_int64),
                                                      C.POINTER(RegResult)]),
    ("kicp_register_staged_sensors_segments", C.c_int, [_P, C.c_int32, _P, C.POINTER(_P), c_dp, c_dp, c_dp, C.c_double,
                                                        C.POINTER(FrameParams), c_dp, c_dp, C.c_int64, C.POINTER(C.c_int64), c_dp, C.c_int64,
                                                        C.POINTER(C.c_int64), C.POINTER(RegResult)]),
    ("kicp_comm_unique_id", C.c_int, [C.POINTER(C.c_uint8)]),
    ("kicp_comm_init", C.c_int, [_P, C.POINTER(C.c_uint8), C.c_int32, C.c_int32]),
    ("kicp_comm_destroy", C.c_int, [_P]),
    ("kicp_comm_p2p_handle", C.c_int, [_P, C.POINTER(C.c_uint8)]),
    ("kicp_comm_p2p_init", C.c_int, [_P, C.POINTER(C.c_uint8), C.c_int32, C.c_int32]),
    ("kicp_register_sharded", C.c_int, [_P, c_dp, C.c_int64, c_dp, c_dp, C.c_double, C.POINTER(RegParams), c_dp,
                                        C.POINTER(RegResult)]),
    ("kicp_register_points_sharded", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, c_dp, c_dp,
                                               C.c_double, C.POINTER(RegParams), c_dp, C.POINTER(RegResult)]),
    ("kicp_register_scan_sharded_async", C.c_int, [_P, _P, c_dp, c_dp, C.c_double, C.POINTER(RegParams),
                                                   C.POINTER(RegResult)]),
]


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("libkicp_b200.so is not built (%s). Run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "or `make -C kinematic-icp_b200/csrc`. There is no CPU fallback." % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _LIB = L
    return _LIB


def check(status, where, allow=(KICP_OK,)):
    if status not in allow:
        raise KicpError(status, where)
    return status


def dp(a):
    return a.ctypes.data_as(c_dp)


def fp(a):
    return a.ctypes.data_as(c_fp)


def as_points(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if a.ndim != 2 or a.shape[1] != 3:
        raise ValueError("expected an (N, 3) array of points")
    return a


def as_cloud(a):
    """(array, dtype code) for an (N, 3) float32 or float64 cloud: float32 stays float32 (half the PCIe bytes)."""
    a = np.asarray(a)
    if a.dtype == np.float32:
        a = np.ascontiguousarray(a)
        code = KICP_DTYPE_F32
    else:
        a = np.ascontiguousarray(a, dtype=np.float64)
        code = KICP_DTYPE_F64
    if a.ndim != 2 or a.shape[1] != 3:
        raise ValueError("expected an (N, 3) array of points")
    return a, code


def as_pose(p):
    return np.ascontiguousarray(p, dtype=np.float64).reshape(7)
