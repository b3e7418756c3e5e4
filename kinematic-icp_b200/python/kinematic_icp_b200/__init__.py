"""H100-native kinematic-icp registration hot path — host-side mirror of the reference's C++ interface.

The classes keep the reference's names and argument meaning:

    kiss_icp::VoxelHashMap                      -> VoxelHashMap       (KISS-ICP v1.2.0 core/VoxelHashMap.hpp)
    kinematic_icp::KinematicRegistration        -> KinematicRegistration  (registration/Registration.hpp:32-50)

Poses are pose7 = [qx, qy, qz, qw, tx, ty, tz] (Sophus::SE3d's two members); point clouds are (N, 3) float64 arrays.
Everything runs on the GPU through libkicp_b200.so (include/kicp.h); there is no CPU fallback.
"""
import ctypes as C

import numpy as np

from . import _capi
from ._capi import (KICP_OK, KICP_WARN_NO_CORRESPONDENCES, KicpError, RegParams, RegResult, as_points, as_pose, check, dp,
                    lib)

__all__ = ["Context", "VoxelHashMap", "Scan", "KinematicRegistration", "KicpError", "RegParams", "RegResult",
           "pinned_empty", "VoxelDownsample", "Preprocess"]


class Context:
    """One GPU: device id, stream, scratch, optional NCCL communicator (kicp_ctx)."""

    def __init__(self, device=0):
        self.h = C.c_void_p()
        check(lib().kicp_ctx_create(int(device), C.byref(self.h)), "kicp_ctx_create")
        self.device = device

    def synchronize(self):
        check(lib().kicp_ctx_synchronize(self.h), "kicp_ctx_synchronize")

    @property
    def stream(self):
        return lib().kicp_ctx_stream(self.h)

    @property
    def launch_count(self):
        return int(lib().kicp_ctx_launch_count(self.h))

    def set_option(self, name, value):
        check(lib().kicp_ctx_set_option(self.h, name.encode(), int(value)), "kicp_ctx_set_option")

    def last_timing(self):
        """Per-pass device timings of the last registration, ns: [pass][certificate phase, its barrier, search phase, barrier
        wait, reduce(+exchange), solve]
        measured on CTA 0 with %globaltimer (kicp_debug_last_timing; synchronises the stream)."""
        L = lib()
        L.kicp_debug_last_timing.argtypes = [C.c_void_p, _capi.c_dp]
        out = np.zeros((_capi.KICP_MAX_ITERATIONS, 6))
        check(L.kicp_debug_last_timing(self.h, dp(out)), "kicp_debug_last_timing")
        return out

    def last_stats(self):
        """(hash probes, candidate points evaluated, 128-byte lines loaded, 0) of the last registration run with option
        "stats" = 1 (kicp_debug_last_stats; synchronises the stream)."""
        L = lib()
        L.kicp_debug_last_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        out = (C.c_uint64 * 4)()
        check(L.kicp_debug_last_stats(self.h, out), "kicp_debug_last_stats")
        return [int(x) for x in out]

    def profile_begin(self):
        check(lib().kicp_ctx_profile_begin(self.h), "kicp_ctx_profile_begin")

    def profile_end(self):
        p = _capi.Profile()
        check(lib().kicp_ctx_profile_end(self.h, C.byref(p)), "kicp_ctx_profile_end")
        return p

    def comm_init(self, unique_id, nranks, rank):
        buf = (C.c_uint8 * _capi.KICP_UNIQUE_ID_BYTES).from_buffer_copy(bytes(unique_id))
        check(lib().kicp_comm_init(self.h, buf, int(nranks), int(rank)), "kicp_comm_init")

    def p2p_handle(self):
        """CUDA-IPC handle of this rank's mailbox (64 bytes) for the fused NVLink exchange."""
        buf = (C.c_uint8 * _capi.KICP_IPC_HANDLE_BYTES)()
        check(lib().kicp_comm_p2p_handle(self.h, buf), "kicp_comm_p2p_handle")
        return bytes(buf)

    def p2p_init(self, handles, nranks, rank):
        """handles: the nranks 64-byte handles in rank order (all-gathered out of band)."""
        blob = b"".join(bytes(h) for h in handles)
        buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        check(lib().kicp_comm_p2p_init(self.h, buf, int(nranks), int(rank)), "kicp_comm_p2p_init")

    def close(self):
        if self.h:
            lib().kicp_ctx_destroy(self.h)
            self.h = C.c_void_p()


def comm_unique_id():
    buf = (C.c_uint8 * _capi.KICP_UNIQUE_ID_BYTES)()
    check(lib().kicp_comm_unique_id(buf), "kicp_comm_unique_id")
    return bytes(buf)


_PINNED = {}


def pinned_empty(shape, dtype=np.float64):
    """numpy array backed by pinned host memory (kicp_host_alloc) so host<->device copies are truly asynchronous."""
    dtype = np.dtype(dtype)
    nbytes = int(np.prod(shape)) * dtype.itemsize
    p = C.c_void_p()
    check(lib().kicp_host_alloc(max(nbytes, 1), C.byref(p)), "kicp_host_alloc")
    buf = (C.c_char * max(nbytes, 1)).from_address(p.value)
    arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
    _PINNED[arr.ctypes.data] = p
    return arr


def pinned_result():
    """A RegResult in pinned host memory, for kicp_register_scan_async."""
    p = C.c_void_p()
    check(lib().kicp_host_alloc(C.sizeof(RegResult), C.byref(p)), "kicp_host_alloc")
    return RegResult.from_address(p.value)


class VoxelHashMap:
    """kiss_icp::VoxelHashMap(voxel_size, max_distance, max_points_per_voxel), resident in HBM."""

    def __init__(self, ctx, voxel_size, max_distance, max_points_per_voxel):
        self.ctx = ctx
        self.voxel_size_, self.max_distance_, self.max_points_per_voxel_ = voxel_size, max_distance, max_points_per_voxel
        self.h = C.c_void_p()
        check(lib().kicp_map_create(ctx.h, float(voxel_size), float(max_distance), int(max_points_per_voxel), C.byref(self.h)),
              "kicp_map_create")

    def close(self):
        if self.h:
            lib().kicp_map_destroy(self.h)
            self.h = C.c_void_p()

    def Clear(self):
        check(lib().kicp_map_clear(self.h), "kicp_map_clear")

    def reserve(self, voxels):
        """Pre-size the device storage (kicp_map_reserve); growth beyond it still works, by doubling."""
        check(lib().kicp_map_reserve(self.h, int(voxels)), "kicp_map_reserve")

    def Empty(self):
        e = C.c_int32()
        check(lib().kicp_map_empty(self.h, C.byref(e)), "kicp_map_empty")
        return bool(e.value)

    def num_points(self):
        n = C.c_int64()
        check(lib().kicp_map_num_points(self.h, C.byref(n)), "kicp_map_num_points")
        return n.value

    def num_voxels(self):
        n = C.c_int64()
        check(lib().kicp_map_num_voxels(self.h, C.byref(n)), "kicp_map_num_voxels")
        return n.value

    def AddPoints(self, points):
        points = as_points(points)
        check(lib().kicp_map_add_points(self.h, dp(points), len(points)), "kicp_map_add_points")

    def RemovePointsFarFromLocation(self, origin):
        o = np.ascontiguousarray(origin, dtype=np.float64).reshape(3)
        check(lib().kicp_map_remove_far(self.h, dp(o)), "kicp_map_remove_far")

    def Update(self, points, origin_or_pose):
        """Update(points, origin) for a 3-vector, Update(points, pose) for a pose7 (KinematicICP.cpp:79)."""
        points = as_points(points)
        a = np.ascontiguousarray(origin_or_pose, dtype=np.float64).ravel()
        if a.size == 3:
            check(lib().kicp_map_update(self.h, dp(points), len(points), dp(a)), "kicp_map_update")
        elif a.size == 7:
            check(lib().kicp_map_update_pose(self.h, dp(points), len(points), dp(a)), "kicp_map_update_pose")
        else:
            raise ValueError("origin (3,) or pose7 (7,) expected")

    def Pointcloud(self):
        n = self.num_points()
        out = np.empty((max(n, 1), 3))
        m = C.c_int64()
        check(lib().kicp_map_pointcloud(self.h, dp(out), n, C.byref(m)), "kicp_map_pointcloud")
        return out[: m.value].copy()

    def export_voxels(self):
        V, n = self.num_voxels(), self.num_points()
        keys = np.empty((max(V, 1), 3), dtype=np.int32)
        counts = np.empty(max(V, 1), dtype=np.int32)
        pts = np.empty((max(n, 1), 3))
        nv, npts = C.c_int64(), C.c_int64()
        check(lib().kicp_map_export_voxels(self.h, keys.ctypes.data_as(_capi.c_ip), counts.ctypes.data_as(_capi.c_ip), dp(pts),
                                           V, n, C.byref(nv), C.byref(npts)), "kicp_map_export_voxels")
        return keys[:V].copy(), counts[:V].copy(), pts[:n].copy()

    def load_voxels(self, keys, counts, points):
        keys = np.ascontiguousarray(keys, dtype=np.int32).reshape(-1, 3)
        counts = np.ascontiguousarray(counts, dtype=np.int32)
        points = as_points(points) if len(points) else np.zeros((0, 3))
        check(lib().kicp_map_load_voxels(self.h, keys.ctypes.data_as(_capi.c_ip), counts.ctypes.data_as(_capi.c_ip), dp(points),
                                         len(counts)), "kicp_map_load_voxels")

    def GetClosestNeighbor(self, queries):
        """Batched GetClosestNeighbor: returns (points (N,3), distances (N,)); (0,0,0), DBL_MAX where nothing is found."""
        q = as_points(queries)
        out = np.empty_like(q)
        d = np.empty(len(q))
        check(lib().kicp_map_nearest(self.h, dp(q), len(q), dp(out), dp(d)), "kicp_map_nearest")
        return out, d


class Scan:
    """A scan resident in HBM (kicp_scan): the `frame` argument of ComputeRobotMotion, uploaded once."""

    def __init__(self, ctx, capacity=0):
        self.ctx = ctx
        self.h = C.c_void_p()
        check(lib().kicp_scan_create(ctx.h, int(capacity), C.byref(self.h)), "kicp_scan_create")

    def upload(self, points, asynchronous=False):
        """float64 or float32 (N, 3): float32 clouds travel and stay as float32, the kernel widens while it reads."""
        points, code = _capi.as_cloud(points)
        self._keepalive = points
        f = lib().kicp_scan_upload_points_async if asynchronous else lib().kicp_scan_upload_points
        check(f(self.h, points.ctypes.data, len(points), code, 0, 0, 0, 0), "kicp_scan_upload_points")

    def close(self):
        if self.h:
            lib().kicp_scan_destroy(self.h)
            self.h = C.c_void_p()


class KinematicRegistration:
    """kinematic_icp::KinematicRegistration (registration/Registration.hpp:32-50).

    max_num_threads is accepted for signature parity and ignored: the GPU path has no thread cap."""

    def __init__(self, max_num_iteration=10, convergence_criterion=1e-3, max_num_threads=1,
                 use_adaptive_odometry_regularization=True, fixed_regularization=0.0):
        self.max_num_iterations_ = max_num_iteration
        self.convergence_criterion_ = convergence_criterion
        self.max_num_threads_ = max_num_threads
        self.use_adaptive_odometry_regularization_ = use_adaptive_odometry_regularization
        self.fixed_regularization_ = fixed_regularization
        self.last_result = None

    def _params(self):
        return RegParams(int(self.max_num_iterations_), int(bool(self.use_adaptive_odometry_regularization_)),
                         float(self.convergence_criterion_), float(self.fixed_regularization_))

    def ComputeRobotMotion(self, frame, voxel_map, last_robot_pose, relative_wheel_odometry, max_correspondence_distance):
        """Host points in, pose7 out (synchronous) — the reference's call at pipeline/KinematicICP.cpp:68-72."""
        frame, code = _capi.as_cloud(frame)
        out = np.empty(7)
        res = RegResult()
        p = self._params()
        if code == _capi.KICP_DTYPE_F64:
            st = lib().kicp_register(voxel_map.h, dp(frame), len(frame), dp(as_pose(last_robot_pose)),
                                     dp(as_pose(relative_wheel_odometry)), float(max_correspondence_distance), C.byref(p), dp(out),
                                     C.byref(res))
        else:
            st = lib().kicp_register_points(voxel_map.h, frame.ctypes.data, len(frame), code, 0, 0, 0, 0, dp(as_pose(last_robot_pose)),
                                            dp(as_pose(relative_wheel_odometry)), float(max_correspondence_distance), C.byref(p),
                                            dp(out), C.byref(res))
        check(st, "kicp_register", allow=(KICP_OK, KICP_WARN_NO_CORRESPONDENCES))
        self.last_result = res
        return out

    def ComputeRobotMotionSharded(self, frame_shard, voxel_map, last_robot_pose, relative_wheel_odometry,
                                  max_correspondence_distance):
        """Every rank passes its contiguous index range of the scan; all ranks return the same pose."""
        frame = as_points(frame_shard)
        out = np.empty(7)
        res = RegResult()
        p = self._params()
        st = lib().kicp_register_sharded(voxel_map.h, dp(frame), len(frame), dp(as_pose(last_robot_pose)),
                                         dp(as_pose(relative_wheel_odometry)), float(max_correspondence_distance), C.byref(p),
                                         dp(out), C.byref(res))
        check(st, "kicp_register_sharded", allow=(KICP_OK, KICP_WARN_NO_CORRESPONDENCES))
        self.last_result = res
        return out

    def enqueue(self, scan, voxel_map, last_robot_pose, relative_wheel_odometry, max_correspondence_distance, result,
                sharded=False):
        """Device-resident scan, no host synchronisation; `result` (pinned_result()) is valid after ctx.synchronize()."""
        p = self._params()
        f = lib().kicp_register_scan_sharded_async if sharded else lib().kicp_register_scan_async
        check(f(voxel_map.h, scan.h, dp(as_pose(last_robot_pose)), dp(as_pose(relative_wheel_odometry)),
                float(max_correspondence_distance), C.byref(p), C.byref(result)), "kicp_register_scan_async")


def VoxelDownsample(ctx, frame, voxel_size):
    """kiss_icp::VoxelDownsample on the device: first point (input order) per voxel, in input order."""
    frame = as_points(frame)
    out = np.empty_like(frame)
    m = C.c_int64()
    check(lib().kicp_voxel_downsample(ctx.h, dp(frame), len(frame), float(voxel_size), dp(out), len(out), C.byref(m)),
          "kicp_voxel_downsample")
    return out[: m.value].copy()


def Preprocess(ctx, frame, timestamps, relative_motion, max_range, min_range, deskew, lidar_to_base=None):
    """kiss_icp::Preprocessor::Preprocess (+ optional transform to the base frame) on the device."""
    frame = as_points(frame)
    ts = np.ascontiguousarray(timestamps, dtype=np.float64)
    ident = np.array([0, 0, 0, 1, 0, 0, 0], dtype=np.float64)
    l2b = ident if lidar_to_base is None else as_pose(lidar_to_base)
    out = np.empty_like(frame)
    m = C.c_int64()
    check(lib().kicp_preprocess(ctx.h, dp(frame), len(frame), dp(ts), len(ts), dp(as_pose(relative_motion)), dp(l2b),
                                float(max_range), float(min_range), int(bool(deskew)), dp(out), len(out), C.byref(m)),
          "kicp_preprocess")
    return out[: m.value].copy()


def RegisterFrame(voxel_map, frame, timestamps, deskew_motion, lidar_to_base, last_pose, relative_odometry, tau, *, max_range=100.0,
                  min_range=0.0, deskew=True, voxel_size=1.0, max_num_iterations=10, convergence_criterion=0.001,
                  use_adaptive_odometry_regularization=True, fixed_regularization=0.0, point_step=0, offsets=(0, 0, 0),
                  want_clouds=True):
    """kicp_register_frame: the per-point part of KinematicICP::RegisterFrame (pipeline/KinematicICP.cpp:48-85) in one call.
    `frame` is float64 [n,3], float32 [n,3], or (with point_step/offsets) a uint8 buffer of PointCloud2-style records with
    float32 x,y,z fields.  Returns (new_pose, preprocessed_frame_in_base, source, result)."""
    from ._capi import KICP_DTYPE_F32, KICP_DTYPE_F64, FrameInput, FrameParams
    inp = FrameInput()
    if point_step:
        raw = np.ascontiguousarray(frame).view(np.uint8).reshape(-1)
        n = raw.size // point_step
        inp.data, inp.n, inp.dtype, inp.point_step = raw.ctypes.data, n, KICP_DTYPE_F32, point_step
        inp.offset_x, inp.offset_y, inp.offset_z = offsets
        keep = raw
    else:
        arr = np.asarray(frame)
        if arr.dtype == np.float32:
            keep = np.ascontiguousarray(arr.reshape(-1, 3))
            inp.dtype = KICP_DTYPE_F32
        else:
            keep = as_points(arr)
            inp.dtype = KICP_DTYPE_F64
        n = len(keep)
        inp.data, inp.n, inp.point_step = keep.ctypes.data, n, 0
    ts = np.ascontiguousarray(timestamps, dtype=np.float64)
    inp.stamps, inp.n_stamps = dp(ts), len(ts)
    fp = FrameParams()
    fp.max_range, fp.min_range, fp.deskew, fp.voxel_size = float(max_range), float(min_range), int(bool(deskew)), float(voxel_size)
    fp.reg.max_num_iterations = int(max_num_iterations)
    fp.reg.use_adaptive_odometry_regularization = int(bool(use_adaptive_odometry_regularization))
    fp.reg.convergence_criterion, fp.reg.fixed_regularization = float(convergence_criterion), float(fixed_regularization)
    out_pose = np.empty(7)
    res = RegResult()
    nf, ns = C.c_int64(), C.c_int64()
    out_frame = np.empty((n, 3)) if want_clouds else None
    out_source = np.empty((n, 3)) if want_clouds else None
    st = lib().kicp_register_frame(voxel_map.h, C.byref(inp), dp(as_pose(deskew_motion)), dp(as_pose(lidar_to_base)), dp(as_pose(last_pose)),
                                   dp(as_pose(relative_odometry)), float(tau), C.byref(fp), dp(out_pose),
                                   dp(out_frame) if want_clouds else None, n, C.byref(nf), dp(out_source) if want_clouds else None, n,
                                   C.byref(ns), C.byref(res))
    if st not in (KICP_OK, KICP_WARN_NO_CORRESPONDENCES):
        check(st, "kicp_register_frame")
    del keep
    if want_clouds:
        return out_pose, out_frame[: nf.value].copy(), out_source[: ns.value].copy(), res
    return out_pose, nf.value, ns.value, res


def shard_range(n, nranks, rank):
    """Contiguous index range [lo, hi) of rank `rank` out of `nranks` (SURVEY.md §8(e))."""
    return n * rank // nranks, n * (rank + 1) // nranks
