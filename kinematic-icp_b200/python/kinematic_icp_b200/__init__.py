"""H100-native kinematic-icp registration hot path — host-side mirror of the reference's C++ interface.

The classes keep the reference's names and argument meaning:

    kiss_icp::VoxelHashMap                      -> VoxelHashMap       (KISS-ICP v1.2.0 core/VoxelHashMap.hpp)
    kinematic_icp::KinematicRegistration        -> KinematicRegistration  (registration/Registration.hpp:32-50)

Poses are pose7 = [qx, qy, qz, qw, tx, ty, tz] (Sophus::SE3d's two members); point clouds are (N, 3) float64 arrays.
Everything runs on the GPU through libkicp_b200.so (include/kicp.h); there is no CPU fallback.
"""
import ctypes as C
import math
from typing import NamedTuple

import numpy as np

from . import _capi, _device
from .deskew import deskew_segments
from ._capi import (KICP_OK, KICP_WARN_NO_CORRESPONDENCES, KicpError, RegParams, RegResult, as_points, as_pose, check, dp,
                    lib)

__all__ = ["Context", "VoxelHashMap", "Scan", "KinematicRegistration", "KicpError", "RegParams", "RegResult",
           "pinned_empty", "VoxelDownsample", "Preprocess",
           "RegisterFrame", "StageFrame", "StageLaserScan", "RegisterStagedFrame", "StagedFrame", "frame_clouds_f32",
           "frame_clouds_device", "PointCloudSensor", "LaserScanSensor", "StageSensors", "StagedSensors", "RegisterStagedSensors",
           "RegisterStagedFrameSegments", "RegisterStagedSensorsSegments", "deskew_segments", "CorrespondenceStats",
           "frame_correspondences", "frame_correspondences_device", "PoseHypothesis", "PlanarAlignment", "frame_map_update",
           "FreeSpaceStats", "frame_free_space", "FREE_SPACE_MIN_MISSES", "FREE_SPACE_END_MARGIN", "OCCUPANCY_INITIAL",
           "OCCUPANCY_HIT_GAIN", "OCCUPANCY_MISS_LOSS", "OCCUPANCY_MAX_EVIDENCE"]

# The defaults of free-space clearing (VoxelHashMap.ClearFreeSpace, Context.set_free_space): see README, "Clearing free space"
FREE_SPACE_MIN_MISSES = 2
FREE_SPACE_END_MARGIN = 0.5
# The defaults of occupancy evidence (VoxelHashMap.set_occupancy): see README, "Clearing free space"
OCCUPANCY_INITIAL = 3
OCCUPANCY_HIT_GAIN = 1
OCCUPANCY_MISS_LOSS = 1
OCCUPANCY_MAX_EVIDENCE = 3


class CorrespondenceStats(NamedTuple):
    """kicp_corr_stats: a cloud's correspondences at a pose.  jtj = (JTJ00, JTJ01, JTJ11) and jtr = (JTr0, JTr1) are
    ComputePerturbation's sums over the inliers before the /N normalisation (the layout of RegResult.sums[:, :5])."""
    n_points: int
    n_inliers: int
    fitness: float
    inlier_rmse: float
    sum_sq: float
    jtj: tuple
    jtr: tuple

    @classmethod
    def from_c(cls, st):
        return cls(int(st.n_points), int(st.n_inliers), float(st.fitness), float(st.inlier_rmse), float(st.sum_sq), tuple(st.jtj),
                   tuple(st.jtr))


class FreeSpaceStats(NamedTuple):
    """kicp_free_space_stats: the rays cast, the voxels visited summed over them, the live voxels and points cleared, and the prior
    voxels that met the clearing condition and were kept."""
    rays: int
    visits: int
    cleared_voxels: int
    cleared_points: int
    prior_contradicted: int

    @classmethod
    def from_c(cls, st):
        return cls(int(st.rays), int(st.visits), int(st.cleared_voxels), int(st.cleared_points), int(st.prior_contradicted))


class PoseHypothesis(NamedTuple):
    """kicp_pose_hypothesis: a pose the pose search scored.  pose = prior * Delta (pose7), offset = (x, y, yaw) of Delta, lattice =
    (ix, iy, ipsi) in units of step / 2^(levels-1), level = the level that scored it."""
    pose: np.ndarray
    offset: tuple
    lattice: tuple
    level: int
    n_inliers: int
    fitness: float
    inlier_rmse: float
    sum_sq: float

    @classmethod
    def from_c(cls, h):
        return cls(np.array(h.pose[:]), tuple(h.offset), tuple(h.lattice), int(h.level), int(h.n_inliers), float(h.fitness),
                   float(h.inlier_rmse), float(h.sum_sq))


class PlanarAlignment(NamedTuple):
    """kicp_planar_alignment: one start's result of VoxelHashMap.AlignPlanar.  pose (pose7) is the returned pose, status one of
    KICP_ALIGN_CONVERGED (0), MAX_ITERATIONS (1), NO_CORRESPONDENCES (2), SINGULAR (3), iterations the updates applied, last_step the
    norm of the last update; the rest is the correspondence report at `pose`: n_inliers, fitness, inlier_rmse, sum_sq, and the
    unnormalised J^T J (00, 01, 02, 11, 12, 22) and J^T r over (x, y, yaw)."""
    pose: np.ndarray
    status: int
    iterations: int
    last_step: float
    n_inliers: int
    fitness: float
    inlier_rmse: float
    sum_sq: float
    jtj: tuple
    jtr: tuple

    @classmethod
    def from_c(cls, a):
        return cls(np.array(a.pose[:]), int(a.status), int(a.iterations), float(a.last_step), int(a.n_inliers), float(a.fitness),
                   float(a.inlier_rmse), float(a.sum_sq), tuple(a.jtj), tuple(a.jtr))


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

    def set_map_update(self, mode, *, min_inliers=0, min_fitness=0.0, max_inlier_rmse=math.inf):
        """kicp_ctx_set_map_update: whether every later frame call on the context ends with the map's Update.  mode is
        _capi.KICP_MAP_UPDATE_ALWAYS (0, default), NEVER (1: register against the map as it is) or GATED (2: update only when the frame's
        correspondence report has n_inliers >= min_inliers, fitness >= min_fitness and inlier_rmse <= max_inlier_rmse, or the map was
        empty).  frame_map_update(ctx) tells what the last frame did."""
        p = _capi.MapUpdatePolicy(int(mode), int(min_inliers), float(min_fitness), float(max_inlier_rmse))
        check(lib().kicp_ctx_set_map_update(self.h, C.byref(p)), "kicp_ctx_set_map_update")

    def set_free_space(self, min_misses=0, end_margin=0.0):
        """kicp_ctx_set_free_space: with min_misses >= 1 the single-sensor frame calls clear free space after every applied Update (the
        rule of VoxelHashMap.ClearFreeSpace on frame_downsample, from lidar_to_base's translation); 0 turns it off.  The multi-sensor
        frame calls refuse to run while it is on.  frame_free_space(ctx) returns the last frame's statistics."""
        p = _capi.FreeSpaceParams(float(end_margin), int(min_misses))
        check(lib().kicp_ctx_set_free_space(self.h, C.byref(p)), "kicp_ctx_set_free_space")

    def wait_stream(self, stream):
        """kicp_ctx_wait_stream: the context's later work waits for everything enqueued on `stream` (a cudaStream_t int) so far."""
        check(lib().kicp_ctx_wait_stream(self.h, stream), "kicp_ctx_wait_stream")

    def stream_wait(self, stream):
        """kicp_stream_wait_ctx: `stream`'s later work waits for everything enqueued on the context so far."""
        check(lib().kicp_stream_wait_ctx(self.h, stream), "kicp_stream_wait_ctx")

    def device_scan(self):
        """The Scan this context keeps for ComputeRobotMotion on device arrays, and the pinned result block it fills."""
        if getattr(self, "_device_scan", None) is None:
            self._device_scan, self._device_result = Scan(self), pinned_result()
        return self._device_scan, self._device_result

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
            if getattr(self, "_device_scan", None) is not None:
                self._device_scan.close()
                self._device_scan = None
            lib().kicp_ctx_destroy(self.h)
            if getattr(self, "_corr_stats", None) is not None:
                self._corr_stats = None
                lib().kicp_host_free(self._corr_stats_mem)
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


_LAYERS = {"all": _capi.KICP_MAP_LAYER_ALL, "prior": _capi.KICP_MAP_LAYER_PRIOR, "live": _capi.KICP_MAP_LAYER_LIVE}


def _layer_code(layer):
    """None (the whole map through the calls without a layer), a KICP_MAP_LAYER_* code, or its name"""
    if layer is None:
        return None
    if isinstance(layer, str):
        if layer not in _LAYERS:
            raise ValueError("layer: one of %s" % ", ".join(sorted(_LAYERS)))
        return _LAYERS[layer]
    return int(layer)


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

    def _device_points(self, points, stream, point_step, offsets):
        """the DevicePoints of a device cloud (see _device.device_points for the accepted layouts), once the context has waited for
        `stream`"""
        d = _device.device_points(points, point_step, offsets)
        self.ctx.wait_stream(_device.resolve_stream(stream, points))
        return d

    def AddPoints(self, points, *, stream=None, point_step=0, offsets=(0, 0, 0)):
        """A device cloud (__cuda_array_interface__: (N, 3) or (N, k) float32 / float64 rows at any row stride, or with point_step
        C-contiguous records with float32 x, y, z at `offsets`) is read on the device after the context has waited for `stream`
        (kicp_map_add_points_device); the call returns when the map is updated."""
        if _device.is_device(points):
            d = self._device_points(points, stream, point_step, offsets)
            check(lib().kicp_map_add_points_device(self.h, d.ptr, d.n, d.dtype, d.point_step, *d.offsets), "kicp_map_add_points_device")
            return
        _host_only("AddPoints", stream=stream, point_step=point_step)
        points = as_points(points)
        check(lib().kicp_map_add_points(self.h, dp(points), len(points)), "kicp_map_add_points")

    def RemovePointsFarFromLocation(self, origin):
        o = np.ascontiguousarray(origin, dtype=np.float64).reshape(3)
        check(lib().kicp_map_remove_far(self.h, dp(o)), "kicp_map_remove_far")

    def Update(self, points, origin_or_pose, *, stream=None, point_step=0, offsets=(0, 0, 0)):
        """Update(points, origin) for a 3-vector, Update(points, pose) for a pose7 (KinematicICP.cpp:79).  A device cloud is taken
        as AddPoints takes it (kicp_map_update_device / kicp_map_update_pose_device)."""
        a = np.ascontiguousarray(origin_or_pose, dtype=np.float64).ravel()
        if a.size not in (3, 7):
            raise ValueError("origin (3,) or pose7 (7,) expected")
        if _device.is_device(points):
            d = self._device_points(points, stream, point_step, offsets)
            f, name = (lib().kicp_map_update_device, "kicp_map_update_device") if a.size == 3 else \
                (lib().kicp_map_update_pose_device, "kicp_map_update_pose_device")
            check(f(self.h, d.ptr, d.n, d.dtype, d.point_step, *d.offsets, dp(a)), name)
            return
        _host_only("Update", stream=stream, point_step=point_step)
        points = as_points(points)
        if a.size == 3:
            check(lib().kicp_map_update(self.h, dp(points), len(points), dp(a)), "kicp_map_update")
        else:
            check(lib().kicp_map_update_pose(self.h, dp(points), len(points), dp(a)), "kicp_map_update_pose")

    def ClearFreeSpace(self, points, pose, sensor_origin=(0.0, 0.0, 0.0), *, min_misses=FREE_SPACE_MIN_MISSES,
                       end_margin=FREE_SPACE_END_MARGIN, stream=None, point_step=0, offsets=(0, 0, 0)):
        """Free-space clearing (kicp_map_clear_free_space): every point of `points` (frame F) is a ray from T * sensor_origin to
        T * p, T = pose (F -> map).  A live voxel that at least `min_misses` rays pass through (each ray cut `end_margin` metres short of
        its end and at max_distance) and in which no ray ends leaves the map; prior voxels are kept and counted.  Returns FreeSpaceStats.
        A device cloud is taken as AddPoints takes it (kicp_map_clear_free_space_device).  The call returns when the map is updated."""
        pose = as_pose(pose)
        o = np.ascontiguousarray(sensor_origin, dtype=np.float64).reshape(3)
        p = _capi.FreeSpaceParams(float(end_margin), int(min_misses))
        st = _capi.FreeSpaceStats()
        if _device.is_device(points):
            d = self._device_points(points, stream, point_step, offsets)
            check(lib().kicp_map_clear_free_space_device(self.h, d.ptr, d.n, d.dtype, d.point_step, *d.offsets, dp(pose), dp(o), C.byref(p),
                                                         C.byref(st)), "kicp_map_clear_free_space_device")
        else:
            _host_only("ClearFreeSpace", stream=stream, point_step=point_step)
            q = as_points(points) if len(points) else np.zeros((0, 3))
            check(lib().kicp_map_clear_free_space(self.h, dp(q), len(q), dp(pose), dp(o), C.byref(p), C.byref(st)),
                  "kicp_map_clear_free_space")
        return FreeSpaceStats.from_c(st)

    def set_occupancy(self, initial=OCCUPANCY_INITIAL, hit_gain=OCCUPANCY_HIT_GAIN, miss_loss=OCCUPANCY_MISS_LOSS,
                      max_evidence=OCCUPANCY_MAX_EVIDENCE):
        """kicp_map_set_occupancy: every live voxel keeps an integer evidence across clearing calls (ClearFreeSpace and the frame
        path's clearing).  A hit adds hit_gain (up to max_evidence); a call in which the voxel is free subtracts miss_loss, and the
        voxel is cleared when its evidence reaches 0.  Every voxel, those in the map now included, starts at `initial`.
        set_occupancy(None) turns it off (memoryless clearing).  The setting belongs to the map: Clear() keeps it."""
        if initial is None:
            check(lib().kicp_map_set_occupancy(self.h, None), "kicp_map_set_occupancy")
            return
        p = _capi.OccupancyParams(int(initial), int(hit_gain), int(miss_loss), int(max_evidence))
        check(lib().kicp_map_set_occupancy(self.h, C.byref(p)), "kicp_map_set_occupancy")

    def occupancy(self):
        """The evidence of every voxel as an np.int32 array aligned with export_voxels() (kicp_map_export_occupancy); raises KicpError
        when occupancy is off."""
        V = self.num_voxels()
        out = np.empty(max(V, 1), dtype=np.int32)
        n = C.c_int64()
        check(lib().kicp_map_export_occupancy(self.h, out.ctypes.data_as(_capi.c_ip), V, C.byref(n)), "kicp_map_export_occupancy")
        return out[: n.value].copy()

    def freeze(self):
        """kicp_map_freeze: every voxel now in the map becomes a read-only prior that Update never evicts and AddPoints never writes
        into; the voxels added later form the live layer beside it.  A second freeze also takes in the live voxels."""
        check(lib().kicp_map_freeze(self.h), "kicp_map_freeze")

    def thaw(self):
        """kicp_map_thaw: the prior becomes ordinary voxels again (the next eviction may remove them)."""
        check(lib().kicp_map_thaw(self.h), "kicp_map_thaw")

    def _prior_size(self):
        v, n = C.c_int64(), C.c_int64()
        check(lib().kicp_map_prior_size(self.h, C.byref(v), C.byref(n)), "kicp_map_prior_size")
        return v.value, n.value

    def num_prior_voxels(self):
        return self._prior_size()[0]

    def num_prior_points(self):
        return self._prior_size()[1]

    def _layer_points(self, layer):
        """the point count of a layer code (None: the whole map); 0 for a code the library refuses"""
        if layer is None or layer == _capi.KICP_MAP_LAYER_ALL:
            return self.num_points()
        n = self._prior_size()[1]
        return {_capi.KICP_MAP_LAYER_PRIOR: n, _capi.KICP_MAP_LAYER_LIVE: self.num_points() - n}.get(layer, 0)

    def _pointcloud(self, layer, dtype):
        n = self._layer_points(layer)
        out = np.empty((max(n, 1), 3), dtype=dtype)
        m = C.c_int64()
        if layer is None:
            if dtype == np.float64:
                check(lib().kicp_map_pointcloud(self.h, dp(out), n, C.byref(m)), "kicp_map_pointcloud")
            else:
                check(lib().kicp_map_pointcloud_f32(self.h, _capi.fp(out), n, C.byref(m)), "kicp_map_pointcloud_f32")
        else:
            code = _capi.KICP_DTYPE_F64 if dtype == np.float64 else _capi.KICP_DTYPE_F32
            check(lib().kicp_map_pointcloud_layer(self.h, int(layer), code, out.ctypes.data, n, C.byref(m)), "kicp_map_pointcloud_layer")
        return out[: m.value].copy()

    def Pointcloud(self, layer=None):
        """Pointcloud(); `layer` (KICP_MAP_LAYER_ALL / _PRIOR / _LIVE, or "all" / "prior" / "live"): one layer of a map with a frozen
        prior (kicp_map_pointcloud_layer), ALL being PRIOR followed by LIVE."""
        return self._pointcloud(_layer_code(layer), np.float64)

    def PointcloudF32(self, layer=None):
        """Pointcloud() as the float32 (N, 3) records EigenToPointCloud2 publishes, narrowed on the device (kicp_map_pointcloud_f32);
        `layer` as for Pointcloud."""
        return self._pointcloud(_layer_code(layer), np.float32)

    def PointcloudInto(self, out, stream=None, layer=None):
        """Pointcloud() (float64 `out`) or PointcloudF32()'s records (float32 `out`) written on the device into `out`, a contiguous
        (cap, 3) device array (__cuda_array_interface__), without a host synchronisation (kicp_map_pointcloud_device_async).  The
        context waits for `stream` first and `stream` waits for the packing after; returns the point count n (rows [0, n) of `out`).
        `layer` as for Pointcloud (kicp_map_pointcloud_layer_device_async)."""
        ptr, cap, code = _device.device_output(out, "PointcloudInto")
        layer = _layer_code(layer)
        s = _device.resolve_stream(stream, out)
        self.ctx.wait_stream(s)
        n = C.c_int64()
        if layer is None:
            check(lib().kicp_map_pointcloud_device_async(self.h, ptr, code, cap, C.byref(n)), "kicp_map_pointcloud_device_async")
        else:
            check(lib().kicp_map_pointcloud_layer_device_async(self.h, layer, code, ptr, cap, C.byref(n)),
                  "kicp_map_pointcloud_layer_device_async")
        self.ctx.stream_wait(s)
        return n.value

    def PointcloudF32Live(self):
        """PointcloudF32()'s records kept up to date incrementally (kicp_map_pointcloud_f32_live): each call writes only the records
        that changed since the previous call into a page-locked buffer the map owns.  Returns (records, stats): records is an (n, 3)
        float32 VIEW of that buffer, in an unspecified order, valid until the next call on this map or close(); stats is a dict of
        added / removed / moved / rewritten / written record counts."""
        rec = _capi.c_fp()
        n = C.c_int64()
        st = _capi.MapLiveStats()
        check(lib().kicp_map_pointcloud_f32_live(self.h, C.byref(rec), C.byref(n), C.byref(st)), "kicp_map_pointcloud_f32_live")
        view = np.ctypeslib.as_array(rec, shape=(max(n.value, 1), 3))[: n.value]
        return view, {f: int(getattr(st, f)) for f, _ in _capi.MapLiveStats._fields_}

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

    def GetClosestNeighbor(self, queries, out=None, stream=None, *, point_step=0, offsets=(0, 0, 0)):
        """Batched GetClosestNeighbor: returns (points (N,3), distances (N,)); (0,0,0), DBL_MAX where nothing is found.

        Device queries (taken as AddPoints takes a device cloud) give device results without a host synchronisation
        (kicp_map_nearest_device_async): the context waits for `stream`, then `stream` waits for the search.  `out` = (points,
        distances), contiguous float64 device arrays of shapes (N, 3) and (N,); without it, torch tensors on the queries' device are
        allocated for torch queries (any other device array needs out).  The queries must stay unchanged until the search has run on
        `stream`."""
        if _device.is_device(queries):
            d = _device.device_points(queries, point_step, offsets)
            if out is None:
                out = (_device.empty_f64(queries, (d.n, 3), "GetClosestNeighbor"), _device.empty_f64(queries, (d.n,), "GetClosestNeighbor"))
            pts, dist = out
            pp = _device.output_f64(pts, (d.n, 3), "GetClosestNeighbor: out[0]")
            pd = _device.output_f64(dist, (d.n,), "GetClosestNeighbor: out[1]")
            s = _device.resolve_stream(stream, queries)
            self.ctx.wait_stream(s)
            check(lib().kicp_map_nearest_device_async(self.h, d.ptr, d.n, d.dtype, d.point_step, *d.offsets, pp, pd),
                  "kicp_map_nearest_device_async")
            self.ctx.stream_wait(s)
            return pts, dist
        _host_only("GetClosestNeighbor", out=out, stream=stream, point_step=point_step)
        q = as_points(queries)
        out = np.empty_like(q)
        d = np.empty(len(q))
        check(lib().kicp_map_nearest(self.h, dp(q), len(q), dp(out), dp(d)), "kicp_map_nearest")
        return out, d


    def Correspondences(self, points, pose, tau, *, out=None, stream=None, point_step=0, offsets=(0, 0, 0)):
        """The correspondences of `points` at `pose` (kicp_map_correspondences): each point moved by the pose, its GetClosestNeighbor,
        the gate distance < tau, and over the inliers the statistics of ComputePerturbation at that pose.  Returns (points (N, 3),
        distances (N,), inlier (N,) uint8, CorrespondenceStats).

        Device points (taken as AddPoints takes a device cloud) give device per-point results (kicp_map_correspondences_device_async):
        the context waits for `stream`, then `stream` waits for the evaluation.  `out` = (points, distances, inlier), contiguous
        float64 (N, 3), float64 (N,) and uint8 (N,) device arrays; without it torch tensors are allocated for torch points (any other
        device array needs out).  The statistics are read back, so the call waits for the evaluation."""
        pose = as_pose(pose)
        tau = float(tau)
        if _device.is_device(points):
            d = _device.device_points(points, point_step, offsets)
            what = "Correspondences"
            if out is None:
                out = (_device.empty_f64(points, (d.n, 3), what), _device.empty_f64(points, (d.n,), what), _device.empty_u8(points, d.n, what))
            pts, dist, inl = out
            pp = _device.output_f64(pts, (d.n, 3), what + ": out[0]")
            pd = _device.output_f64(dist, (d.n,), what + ": out[1]")
            pi = _device.output_u8(inl, d.n, what + ": out[2]")
            s = _device.resolve_stream(stream, points)
            self.ctx.wait_stream(s)
            st = _pinned_corr_stats(self.ctx)
            check(lib().kicp_map_correspondences_device_async(self.h, d.ptr, d.n, d.dtype, d.point_step, *d.offsets, dp(pose), tau, pp, pd,
                                                              pi, C.addressof(st)), "kicp_map_correspondences_device_async")
            self.ctx.stream_wait(s)
            self.ctx.synchronize()
            return pts, dist, inl, CorrespondenceStats.from_c(st)
        _host_only("Correspondences", out=out, stream=stream, point_step=point_step)
        q = as_points(points)
        pts, dist, inl = np.empty_like(q), np.empty(len(q)), np.empty(len(q), np.uint8)
        st = _capi.CorrStats()
        check(lib().kicp_map_correspondences(self.h, dp(q), len(q), dp(pose), tau, dp(pts), dp(dist), inl.ctypes.data, C.byref(st)),
              "kicp_map_correspondences")
        return pts, dist, inl, CorrespondenceStats.from_c(st)

    def PoseSearch(self, points, prior, tau, half_extent, step, levels=3, keep=8, *, stream=None, point_step=0, offsets=(0, 0, 0)):
        """Where `points` (robot base frame) fit the map around `prior` (kicp_map_pose_search): a lattice of planar offsets (x, y,
        yaw) of +-half_extent on `step` scored at level 0, then the 26 neighbours of the `keep` best at each finer level (step / 2^l).
        A hypothesis's score is Correspondences(points, pose, tau)'s inlier count (exactly) and its sum of squared distances (to
        rounding: it is added in an order of its own).  Returns (the best
        min(keep, n_scored) as PoseHypothesis, best first; n_scored).  The map is not modified.

        Device points (taken as AddPoints takes a device cloud) are read on the device (kicp_map_pose_search_device) after the
        context has waited for `stream`."""
        prior = as_pose(prior)
        p = _capi.PoseSearchParams((C.c_double * 3)(*[float(v) for v in half_extent]), (C.c_double * 3)(*[float(v) for v in step]),
                                   float(tau), int(levels), int(keep))
        cap = max(int(keep), 1)
        out = (_capi.PoseHypothesis * cap)()
        n_out, n_scored = C.c_int32(), C.c_int64()
        if _device.is_device(points):
            d = self._device_points(points, stream, point_step, offsets)
            check(lib().kicp_map_pose_search_device(self.h, d.ptr, d.n, d.dtype, d.point_step, *d.offsets, dp(prior), C.byref(p), out,
                                                    cap, C.byref(n_out), C.byref(n_scored)), "kicp_map_pose_search_device")
        else:
            _host_only("PoseSearch", stream=stream, point_step=point_step)
            q = as_points(points) if len(points) else np.zeros((0, 3))
            check(lib().kicp_map_pose_search(self.h, dp(q), len(q), dp(prior), C.byref(p), out, cap, C.byref(n_out),
                                             C.byref(n_scored)), "kicp_map_pose_search")
        return [PoseHypothesis.from_c(out[i]) for i in range(n_out.value)], n_scored.value

    def AlignPlanar(self, points, initial, tau, max_iterations=10, convergence=1e-3, *, stream=None, point_step=0, offsets=(0, 0, 0)):
        """Gauss-Newton in (x, y, yaw) of `points` (robot base frame) against the map from each starting pose of `initial` (one
        pose7, or a (k, 7) array-like of 1 to 64 poses, each aligned on its own; kicp_map_align_planar): at most `max_iterations`
        updates T = T * Delta(dx) over the inliers d < tau, stopping when |dx| < convergence (the defaults are the reference's
        max_num_iterations and convergence_criterion).  Returns one PlanarAlignment per start, in input order, with the report taken
        at the returned pose.  One host synchronisation; the map is not modified.

        Device points (taken as AddPoints takes a device cloud) are read on the device (kicp_map_align_planar_device) after the
        context has waited for `stream`."""
        starts = np.ascontiguousarray(initial, dtype=np.float64)
        if starts.ndim not in (1, 2) or starts.shape[-1] != 7:
            raise ValueError("initial: expected one pose7 or a (k, 7) array of poses")
        starts = starts.reshape(-1, 7)
        k = len(starts)
        p = _capi.PlanarAlignParams(float(tau), float(convergence), int(max_iterations))
        out = (_capi.PlanarAlignment * max(k, 1))()
        if _device.is_device(points):
            d = self._device_points(points, stream, point_step, offsets)
            check(lib().kicp_map_align_planar_device(self.h, d.ptr, d.n, d.dtype, d.point_step, *d.offsets, dp(starts), k, C.byref(p),
                                                     out), "kicp_map_align_planar_device")
        else:
            _host_only("AlignPlanar", stream=stream, point_step=point_step)
            q = as_points(points) if len(points) else np.zeros((0, 3))
            check(lib().kicp_map_align_planar(self.h, dp(q), len(q), dp(starts), k, C.byref(p), out), "kicp_map_align_planar")
        return [PlanarAlignment.from_c(out[i]) for i in range(k)]


def _pinned_corr_stats(ctx):
    """a CorrStats in page-locked memory the context keeps (the stats of kicp_map_correspondences_device_async)"""
    if getattr(ctx, "_corr_stats", None) is None:
        p = C.c_void_p()
        check(lib().kicp_host_alloc(C.sizeof(_capi.CorrStats), C.byref(p)), "kicp_host_alloc")
        ctx._corr_stats_mem = p
        ctx._corr_stats = _capi.CorrStats.from_address(p.value)
    return ctx._corr_stats


def frame_correspondences(ctx):
    """CorrespondenceStats of the last frame registered on `ctx` with option "correspondences" 1 (kicp_frame_correspondences): its
    registration source at the returned pose against the map before the frame's Update.  All zero when the option was off or the
    frame failed."""
    st = _capi.CorrStats()
    check(lib().kicp_frame_correspondences(ctx.h, C.byref(st)), "kicp_frame_correspondences")
    return CorrespondenceStats.from_c(st)


def frame_map_update(ctx):
    """The map-update outcome of the last frame call on `ctx` (kicp_frame_map_update): _capi.KICP_FRAME_UPDATE_APPLIED (0),
    NO_CORRESPONDENCES (1), REJECTED (2), SKIPPED (3), or NONE (4) before the first frame, after a frame that failed, and after any other
    front-end call."""
    o = C.c_int32()
    check(lib().kicp_frame_map_update(ctx.h, C.byref(o)), "kicp_frame_map_update")
    return int(o.value)


def frame_free_space(ctx):
    """FreeSpaceStats of the last frame call on `ctx` (kicp_frame_free_space): all zero when the option was off, the Update was not
    applied or the frame failed."""
    st = _capi.FreeSpaceStats()
    check(lib().kicp_frame_free_space(ctx.h, C.byref(st)), "kicp_frame_free_space")
    return FreeSpaceStats.from_c(st)


def frame_correspondences_device(ctx):
    """(points (n, 3) float64, distances (n,) float64, inlier (n,) uint8) of that evaluation, one row per source point, zero-copy in
    context-owned device memory (kicp_frame_correspondences_device), with frame_clouds_device's lifetime: copy them to keep them."""
    pp, pd, pi = C.c_void_p(), C.c_void_p(), C.c_void_p()
    n = C.c_int64()
    check(lib().kicp_frame_correspondences_device(ctx.h, C.byref(pp), C.byref(pd), C.byref(pi), C.byref(n)),
          "kicp_frame_correspondences_device")
    return (_device.DeviceArray(pp.value, (n.value, 3), "<f8", ctx), _device.DeviceArray(pd.value, (n.value,), "<f8", ctx),
            _device.DeviceArray(pi.value, (n.value,), "|u1", ctx))


class Scan:
    """A scan resident in HBM (kicp_scan): the `frame` argument of ComputeRobotMotion, uploaded once."""

    def __init__(self, ctx, capacity=0):
        self.ctx = ctx
        self.h = C.c_void_p()
        check(lib().kicp_scan_create(ctx.h, int(capacity), C.byref(self.h)), "kicp_scan_create")

    def upload(self, points, asynchronous=False, stream=None):
        """float64 or float32 (N, 3): float32 clouds travel and stay as float32, the kernel widens while it reads.  A device array
        (__cuda_array_interface__, rows of (N, k) float32 / float64 at any row stride) is attached instead (kicp_scan_attach_device):
        the registrations read it in place, after the context has waited for `stream`; the scan keeps it alive until the next
        upload, and it must stay unchanged until those registrations have completed."""
        if _device.is_device(points):
            d = _device.device_points(points)
            self.ctx.wait_stream(_device.resolve_stream(stream, points))
            check(lib().kicp_scan_attach_device(self.h, d.ptr, d.n, d.dtype, d.point_step, *d.offsets), "kicp_scan_attach_device")
            self._keepalive = points
            return
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

    def ComputeRobotMotion(self, frame, voxel_map, last_robot_pose, relative_wheel_odometry, max_correspondence_distance,
                           stream=None):
        """Host points in, pose7 out (synchronous) — the reference's call at pipeline/KinematicICP.cpp:68-72.  A device `frame`
        (__cuda_array_interface__) is attached to a scan the map's Context keeps and registered in place, after the context has waited
        for `stream`; the call returns when the registration has completed."""
        if _device.is_device(frame):
            scan, res = voxel_map.ctx.device_scan()
            scan.upload(frame, stream=stream)
            p = self._params()
            st = lib().kicp_register_scan_async(voxel_map.h, scan.h, dp(as_pose(last_robot_pose)), dp(as_pose(relative_wheel_odometry)),
                                                float(max_correspondence_distance), C.byref(p), C.byref(res))
            check(st, "kicp_register_scan_async")
            voxel_map.ctx.synchronize()
            self.last_result = RegResult.from_buffer_copy(res)
            check(self.last_result.status, "kicp_register_scan_async", allow=(KICP_OK, KICP_WARN_NO_CORRESPONDENCES))
            return self.last_result.pose_np()
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


def _host_only(what, **device_keywords):
    """A host input takes none of the keywords of the device path (out=, stream=, point_step=): ValueError if one is given."""
    given = [k for k, v in device_keywords.items() if v is not None and v != 0]
    if given:
        raise ValueError("%s: %s apply to device inputs only" % (what, ", ".join(given)))


def _device_frontend_out(frame, n, out, what):
    """(out, pointer, capacity) of the output of a device front-end call: `out`, a contiguous (cap, 3) float64 device array, or a new
    (n, 3) torch tensor for a torch frame"""
    if out is None:
        out = _device.empty_f64(frame, (n, 3), what)
    ptr, cap, code = _device.device_output(out, what + ": out")
    if code != _capi.KICP_DTYPE_F64:
        raise ValueError("%s: out must be float64" % what)
    return out, ptr, cap


def VoxelDownsample(ctx, frame, voxel_size, *, out=None, stream=None, point_step=0, offsets=(0, 0, 0)):
    """kiss_icp::VoxelDownsample on the device: first point (input order) per voxel, in input order; after
    ctx.set_option("downsample_order", 1), in the iteration order of KISS-ICP's robin_map (include/kicp.h; unpinned).

    A device `frame` (taken as VoxelHashMap.AddPoints takes a device cloud) is read after the context has waited for `stream`
    (kicp_voxel_downsample_device); the survivors go to `out`, a contiguous (cap, 3) float64 device array (a new torch tensor of n
    rows for a torch frame when omitted), and the call returns out[:m] once they are there."""
    if _device.is_device(frame):
        d = _device.device_points(frame, point_step, offsets)
        out, ptr, cap = _device_frontend_out(frame, d.n, out, "VoxelDownsample")
        ctx.wait_stream(_device.resolve_stream(stream, frame))
        m = C.c_int64()
        check(lib().kicp_voxel_downsample_device(ctx.h, d.ptr, d.n, d.dtype, d.point_step, *d.offsets, float(voxel_size), ptr, cap,
                                                 C.byref(m)), "kicp_voxel_downsample_device")
        return out[: m.value]
    _host_only("VoxelDownsample", out=out, stream=stream, point_step=point_step)
    frame = as_points(frame)
    out = np.empty_like(frame)
    m = C.c_int64()
    check(lib().kicp_voxel_downsample(ctx.h, dp(frame), len(frame), float(voxel_size), dp(out), len(out), C.byref(m)),
          "kicp_voxel_downsample")
    return out[: m.value].copy()


def Preprocess(ctx, frame, timestamps, relative_motion, max_range, min_range, deskew, lidar_to_base=None, *, out=None, stream=None,
               point_step=0, offsets=(0, 0, 0)):
    """kiss_icp::Preprocessor::Preprocess (+ optional transform to the base frame) on the device.

    A device `frame` is taken as VoxelDownsample takes one (kicp_preprocess_device); its timestamps, if any, are then a 1-D float64
    device array."""
    ident = np.array([0, 0, 0, 1, 0, 0, 0], dtype=np.float64)
    l2b = ident if lidar_to_base is None else as_pose(lidar_to_base)
    if _device.is_device(frame):
        inp, n = _device_frame_input(frame, timestamps, point_step, offsets)
        out, ptr, cap = _device_frontend_out(frame, n, out, "Preprocess")
        ctx.wait_stream(_device.resolve_stream(stream, frame))
        m = C.c_int64()
        check(lib().kicp_preprocess_device(ctx.h, inp.data, inp.n, inp.dtype, inp.point_step, inp.offset_x, inp.offset_y, inp.offset_z,
                                           C.cast(inp.stamps, C.c_void_p), inp.n_stamps, dp(as_pose(relative_motion)), dp(l2b),
                                           float(max_range), float(min_range), int(bool(deskew)), ptr, cap, C.byref(m)),
              "kicp_preprocess_device")
        return out[: m.value]
    if _device.is_device(timestamps):
        raise ValueError("a host frame takes its timestamps from host memory")
    _host_only("Preprocess", out=out, stream=stream, point_step=point_step)
    frame = as_points(frame)
    ts = np.ascontiguousarray(timestamps, dtype=np.float64)
    out = np.empty_like(frame)
    m = C.c_int64()
    check(lib().kicp_preprocess(ctx.h, dp(frame), len(frame), dp(ts), len(ts), dp(as_pose(relative_motion)), dp(l2b),
                                float(max_range), float(min_range), int(bool(deskew)), dp(out), len(out), C.byref(m)),
          "kicp_preprocess")
    return out[: m.value].copy()


def _frame_input(frame, timestamps, point_step, offsets):
    """(kicp_frame_input, buffers to keep alive, n) for RegisterFrame / StageFrame"""
    from ._capi import KICP_DTYPE_F32, KICP_DTYPE_F64, FrameInput
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
    return inp, (keep, ts), n


def _frame_params(max_range, min_range, deskew, voxel_size, max_num_iterations, convergence_criterion,
                  use_adaptive_odometry_regularization, fixed_regularization):
    from ._capi import FrameParams
    fp = FrameParams()
    fp.max_range, fp.min_range, fp.deskew, fp.voxel_size = float(max_range), float(min_range), int(bool(deskew)), float(voxel_size)
    fp.reg.max_num_iterations = int(max_num_iterations)
    fp.reg.use_adaptive_odometry_regularization = int(bool(use_adaptive_odometry_regularization))
    fp.reg.convergence_criterion, fp.reg.fixed_regularization = float(convergence_criterion), float(fixed_regularization)
    return fp


def _register(f, args, n, want_clouds, where, ctx=None):
    """kicp_register_frame / kicp_register_staged_frame with output buffers of n points: (new_pose, frame, source, result).  With
    `ctx` (f32_clouds) the clouds are the float32 records of kicp_frame_clouds_f32 instead, and no double buffers are passed."""
    out_pose = np.empty(7)
    res = RegResult()
    nf, ns = C.c_int64(), C.c_int64()
    want_f64 = want_clouds and ctx is None
    out_frame = np.empty((n, 3)) if want_f64 else None
    out_source = np.empty((n, 3)) if want_f64 else None
    st = f(*args, dp(out_pose), dp(out_frame) if want_f64 else None, n, C.byref(nf), dp(out_source) if want_f64 else None, n,
           C.byref(ns), C.byref(res))
    if st not in (KICP_OK, KICP_WARN_NO_CORRESPONDENCES):
        check(st, where)
    if ctx is not None:
        return (out_pose,) + frame_clouds_f32(ctx) + (res,)
    if want_clouds:
        return out_pose, out_frame[: nf.value].copy(), out_source[: ns.value].copy(), res
    return out_pose, nf.value, ns.value, res


def frame_clouds_f32(ctx):
    """(frame, source) of the last frame registered on `ctx` with KICP_STAGE_F32, as float32 (N, 3) copies (kicp_frame_clouds_f32)."""
    pf, ps = _capi.c_fp(), _capi.c_fp()
    nf, ns = C.c_int64(), C.c_int64()
    check(lib().kicp_frame_clouds_f32(ctx.h, C.byref(pf), C.byref(nf), C.byref(ps), C.byref(ns)), "kicp_frame_clouds_f32")
    frame = np.ctypeslib.as_array(pf, shape=(nf.value, 3)).copy() if nf.value else np.zeros((0, 3), np.float32)
    source = np.ctypeslib.as_array(ps, shape=(ns.value, 3)).copy() if ns.value else np.zeros((0, 3), np.float32)
    return frame, source


def frame_clouds_device(ctx, dtype=_capi.KICP_DTYPE_F64):
    """(frame, source) of the last frame registered on `ctx`, zero-copy in context-owned device memory (kicp_frame_clouds_device):
    objects exposing __cuda_array_interface__ for torch.as_tensor / cupy.asarray, (n, 3) float64 (KICP_DTYPE_F64) or the float32
    records of a KICP_STAGE_F32 frame (KICP_DTYPE_F32).  Valid until the next front-end call on `ctx`; copy them to keep them."""
    pf, ps = C.c_void_p(), C.c_void_p()
    nf, ns = C.c_int64(), C.c_int64()
    check(lib().kicp_frame_clouds_device(ctx.h, int(dtype), C.byref(pf), C.byref(nf), C.byref(ps), C.byref(ns)),
          "kicp_frame_clouds_device")
    return _device.DeviceCloud(pf.value, nf.value, dtype, ctx), _device.DeviceCloud(ps.value, ns.value, dtype, ctx)


def RegisterFrame(voxel_map, frame, timestamps, deskew_motion, lidar_to_base, last_pose, relative_odometry, tau, *, max_range=100.0,
                  min_range=0.0, deskew=True, voxel_size=1.0, max_num_iterations=10, convergence_criterion=0.001,
                  use_adaptive_odometry_regularization=True, fixed_regularization=0.0, point_step=0, offsets=(0, 0, 0),
                  want_clouds=True, f32_clouds=False):
    """kicp_register_frame: the per-point part of KinematicICP::RegisterFrame (pipeline/KinematicICP.cpp:48-85) in one call.
    `frame` is float64 [n,3], float32 [n,3], or (with point_step/offsets) a uint8 buffer of PointCloud2-style records with
    float32 x,y,z fields.  Returns (new_pose, preprocessed_frame_in_base, source, result); with f32_clouds the two clouds are the
    float32 records a node publishes (KICP_STAGE_F32, kicp_frame_clouds_f32).  Both down-samples follow the context's option
    "downsample_order" (ctx.set_option("downsample_order", 1): KISS-ICP's robin_map order); nothing else is needed."""
    inp, keep, n = _frame_input(frame, timestamps, point_step, offsets)
    fp = _frame_params(max_range, min_range, deskew, voxel_size, max_num_iterations, convergence_criterion,
                       use_adaptive_odometry_regularization, fixed_regularization)
    if f32_clouds:
        fp.stage_clouds = _capi.KICP_STAGE_F32
    args = (voxel_map.h, C.byref(inp), dp(as_pose(deskew_motion)), dp(as_pose(lidar_to_base)), dp(as_pose(last_pose)),
            dp(as_pose(relative_odometry)), float(tau), C.byref(fp))
    out = _register(lib().kicp_register_frame, args, n, want_clouds, "kicp_register_frame", voxel_map.ctx if f32_clouds else None)
    del keep
    return out


class StagedFrame(NamedTuple):
    """What StageFrame returns: the frame's point count, the stamps' [min, max] in seconds and their count (0: no stamps)."""
    n: int
    stamp_range: np.ndarray
    n_stamps: int


def _device_frame_input(frame, timestamps, point_step, offsets):
    """kicp_frame_input of a device frame (and device stamps, if any): see _device.device_points for the accepted layouts"""
    from ._capi import FrameInput
    if len(timestamps) and not _device.is_device(timestamps):
        raise ValueError("a device frame takes its timestamps as a device array too")
    d = _device.device_points(frame, point_step, offsets)
    inp = FrameInput()
    inp.data, inp.n, inp.dtype, inp.point_step = d.ptr or None, d.n, d.dtype, d.point_step
    inp.offset_x, inp.offset_y, inp.offset_z = d.offsets
    if len(timestamps):
        ptr, inp.n_stamps = _device.device_vector(timestamps, "<f8", "timestamps")
        inp.stamps = C.cast(C.c_void_p(ptr), _capi.c_dp)
    return inp, d.n


def StageFrame(ctx, frame, *, point_step=0, offsets=(0, 0, 0), stamp_datatype=0, stamp_offset=0, timestamps=(), stream=None):
    """kicp_frame_stage: upload `frame` (as RegisterFrame takes it) once and decode its points and, with stamp_datatype 6 / 7 / 8
    (PointField UINT32 / FLOAT32 / FLOAT64), the time field at byte `stamp_offset` of every record on the device; the frame waits
    there for RegisterStagedFrame.  Returns a StagedFrame; SweepTiming follows from its stamp_range (kicp/pointcloud2.hpp
    sweep_timing).

    A `frame` exposing __cuda_array_interface__ is staged from device memory instead (kicp_frame_stage_device, read in place after
    the context has waited for `stream`): (N, 3) or (N, k) float32 / float64 rows at any row stride, or with point_step C-contiguous
    records; timestamps, if any, are then a 1-D float64 device array."""
    if _device.is_device(frame):
        inp, n = _device_frame_input(frame, timestamps, point_step, offsets)
        ctx.wait_stream(_device.resolve_stream(stream, frame))
        rng, ns = np.zeros(2), C.c_int64()
        check(lib().kicp_frame_stage_device(ctx.h, C.byref(inp), int(stamp_datatype), int(stamp_offset), dp(rng), C.byref(ns)),
              "kicp_frame_stage_device")
        return StagedFrame(n, rng, ns.value)
    if _device.is_device(timestamps):
        raise ValueError("a host frame takes its timestamps from host memory")
    inp, keep, n = _frame_input(frame, timestamps, point_step, offsets)
    rng, ns = np.zeros(2), C.c_int64()
    check(lib().kicp_frame_stage(ctx.h, C.byref(inp), int(stamp_datatype), int(stamp_offset), dp(rng), C.byref(ns)), "kicp_frame_stage")
    del keep
    return StagedFrame(n, rng, ns.value)


def StageLaserScan(ctx, ranges, *, angle_min, angle_max, angle_increment, time_increment, range_min, range_max, stream=None):
    """kicp_frame_stage_laser_scan: a sensor_msgs/LaserScan staged as the frame laser_geometry's projectLaser makes of it (points in
    the scan plane, per-beam stamps); the ranges cross PCIe once.  Returns a StagedFrame whose n and n_stamps are the kept beam
    count; RegisterStagedFrame registers it.  Ranges exposing __cuda_array_interface__ (1-D contiguous float32) are read in place
    instead (kicp_frame_stage_laser_scan_device), after the context has waited for `stream`."""
    if _device.is_device(ranges):
        ptr, n = _device.device_vector(ranges, "<f4", "ranges")
        f, where = lib().kicp_frame_stage_laser_scan_device, "kicp_frame_stage_laser_scan_device"
        ctx.wait_stream(_device.resolve_stream(stream, ranges))
        r, rp = ranges, C.cast(C.c_void_p(ptr), _capi.c_fp)
    else:
        r = np.ascontiguousarray(ranges, dtype=np.float32).reshape(-1)
        f, where, n, rp = lib().kicp_frame_stage_laser_scan, "kicp_frame_stage_laser_scan", len(r), _capi.fp(r)
    scan = _capi.LaserScan(rp, n, angle_min, angle_max, angle_increment, time_increment, range_min, range_max)
    rng, m = np.zeros(2), C.c_int64()
    check(f(ctx.h, C.byref(scan), dp(rng), C.byref(m)), where)
    del r
    return StagedFrame(m.value, rng, m.value)


def RegisterStagedFrame(voxel_map, staged, deskew_motion, lidar_to_base, last_pose, relative_odometry, tau, *, max_range=100.0,
                        min_range=0.0, deskew=True, voxel_size=1.0, max_num_iterations=10, convergence_criterion=0.001,
                        use_adaptive_odometry_regularization=True, fixed_regularization=0.0, want_clouds=True, f32_clouds=False):
    """kicp_register_staged_frame: RegisterFrame on the frame StageFrame left on voxel_map's context (`staged` = its StagedFrame).
    Same results as RegisterFrame given the same points and the host-decoded stamps; f32_clouds and the context's option
    "downsample_order" as there."""
    fp = _frame_params(max_range, min_range, deskew, voxel_size, max_num_iterations, convergence_criterion,
                       use_adaptive_odometry_regularization, fixed_regularization)
    if f32_clouds:
        fp.stage_clouds = _capi.KICP_STAGE_F32
    args = (voxel_map.h, dp(as_pose(deskew_motion)), dp(as_pose(lidar_to_base)), dp(as_pose(last_pose)), dp(as_pose(relative_odometry)),
            float(tau), C.byref(fp))
    return _register(lib().kicp_register_staged_frame, args, staged.n, want_clouds, "kicp_register_staged_frame",
                     voxel_map.ctx if f32_clouds else None)


class PointCloudSensor:
    """One sensor of StageSensors: a frame as StageFrame takes it (host, or __cuda_array_interface__ with device timestamps) and the
    seconds added to its stamps to put them on the frame's common clock (0 for absolute stamps, the header stamp for relative ones)."""

    def __init__(self, frame, *, point_step=0, offsets=(0, 0, 0), stamp_datatype=0, stamp_offset=0, timestamps=(), time_offset=0.0):
        if not np.isfinite(time_offset):
            raise ValueError("time_offset must be finite")
        if len(timestamps) and not _device.is_device(timestamps) and not _device.is_device(frame) and not point_step:
            if len(timestamps) != len(np.asarray(frame).reshape(-1, 3)):
                raise ValueError("timestamps must hold one stamp per point")
        self.frame, self.point_step, self.offsets = frame, int(point_step), tuple(offsets)
        self.stamp_datatype, self.stamp_offset, self.timestamps, self.time_offset = int(stamp_datatype), int(stamp_offset), timestamps, float(time_offset)


class LaserScanSensor:
    """One sensor of StageSensors: a LaserScan as StageLaserScan takes it and its header stamp as time_offset (its beam times are
    relative to it)."""

    def __init__(self, ranges, *, angle_min, angle_max, angle_increment, time_increment, range_min, range_max, time_offset=0.0):
        if not np.isfinite(time_offset):
            raise ValueError("time_offset must be finite")
        self.ranges, self.angle_min, self.angle_max, self.angle_increment = ranges, angle_min, angle_max, angle_increment
        self.time_increment, self.range_min, self.range_max, self.time_offset = time_increment, range_min, range_max, float(time_offset)


class StagedSensors(NamedTuple):
    """What StageSensors returns: the staged points of all sensors, the common window [T0, T1] in seconds and the stamp count (0: no
    sensor has stamps), the sensor count, and per sensor (n_points, n_stamps, stamp_range on the common clock)."""
    n: int
    stamp_range: np.ndarray
    n_stamps: int
    k: int
    sensors: tuple


def StageSensors(ctx, sensors, stream=None):
    """kicp_frame_stage_sensors: stage the frame of several LiDARs (PointCloudSensor / LaserScanSensor, each from host memory or
    __cuda_array_interface__ objects) with one host synchronisation; RegisterStagedSensors registers it.  Device inputs are read in place
    after the context has waited for `stream`."""
    sensors = list(sensors)
    if not 1 <= len(sensors) <= _capi.KICP_MAX_SENSORS:
        raise ValueError("StageSensors takes 1 to %d sensors" % _capi.KICP_MAX_SENSORS)
    arr = (_capi.SensorInput * len(sensors))()
    keep, producer = [], None
    for i, sen in enumerate(sensors):
        d = arr[i]
        d.time_offset = sen.time_offset if isinstance(sen, (PointCloudSensor, LaserScanSensor)) else 0.0
        if isinstance(sen, PointCloudSensor):
            d.kind, d.stamp_datatype, d.stamp_offset = _capi.KICP_SENSOR_POINTS, sen.stamp_datatype, sen.stamp_offset
            if _device.is_device(sen.frame):
                d.points, _ = _device_frame_input(sen.frame, sen.timestamps, sen.point_step, sen.offsets)
                d.device = 1
                producer = sen.frame if producer is None else producer
                keep.append(sen.timestamps)
            else:
                if _device.is_device(sen.timestamps):
                    raise ValueError("a host frame takes its timestamps from host memory")
                d.points, buf, _ = _frame_input(sen.frame, sen.timestamps, sen.point_step, sen.offsets)
                keep.append(buf)
        elif isinstance(sen, LaserScanSensor):
            d.kind = _capi.KICP_SENSOR_LASER_SCAN
            if _device.is_device(sen.ranges):
                ptr, n = _device.device_vector(sen.ranges, "<f4", "ranges")
                d.device, rp = 1, C.cast(C.c_void_p(ptr), _capi.c_fp)
                producer = sen.ranges if producer is None else producer
            else:
                r = np.ascontiguousarray(sen.ranges, dtype=np.float32).reshape(-1)
                keep.append(r)
                n, rp = len(r), _capi.fp(r)
            d.scan = _capi.LaserScan(rp, n, sen.angle_min, sen.angle_max, sen.angle_increment, sen.time_increment, sen.range_min, sen.range_max)
        else:
            raise TypeError("sensor %d is neither a PointCloudSensor nor a LaserScanSensor" % i)
    if producer is not None:
        ctx.wait_stream(_device.resolve_stream(stream, producer))
    rng, stats = np.zeros(2), (_capi.SensorStats * len(sensors))()
    check(lib().kicp_frame_stage_sensors(ctx.h, arr, len(sensors), dp(rng), stats), "kicp_frame_stage_sensors")
    del keep
    per = tuple((st.n_points, st.n_stamps, np.array(st.stamp_range[:])) for st in stats)
    return StagedSensors(sum(p[0] for p in per), rng, sum(p[1] for p in per), len(sensors), per)


def RegisterStagedSensors(voxel_map, staged, deskew_motions, lidar_to_bases, last_pose, relative_odometry, tau, *, max_range=100.0,
                          min_range=0.0, deskew=True, voxel_size=1.0, max_num_iterations=10, convergence_criterion=0.001,
                          use_adaptive_odometry_regularization=True, fixed_regularization=0.0, want_clouds=True, f32_clouds=False):
    """kicp_register_staged_sensors: RegisterFrame on the frame StageSensors left on voxel_map's context (`staged` = its StagedSensors,
    or the StagedFrame of a single-sensor staging call), sensor i de-skewed with deskew_motions[i] and moved to base by lidar_to_bases[i].
    Returns what RegisterStagedFrame returns."""
    motions = np.ascontiguousarray([as_pose(p) for p in deskew_motions], dtype=np.float64).reshape(-1, 7)
    l2bs = np.ascontiguousarray([as_pose(p) for p in lidar_to_bases], dtype=np.float64).reshape(-1, 7)
    k = getattr(staged, "k", 1)  # a StagedFrame of StageFrame / StageLaserScan is one sensor
    if len(motions) != k or len(l2bs) != k:
        raise ValueError("one deskew motion and one lidar_to_base per staged sensor (%d)" % k)
    fp = _frame_params(max_range, min_range, deskew, voxel_size, max_num_iterations, convergence_criterion,
                       use_adaptive_odometry_regularization, fixed_regularization)
    if f32_clouds:
        fp.stage_clouds = _capi.KICP_STAGE_F32
    args = (voxel_map.h, k, dp(motions), dp(l2bs), dp(as_pose(last_pose)), dp(as_pose(relative_odometry)), float(tau), C.byref(fp))
    return _register(lib().kicp_register_staged_sensors, args, staged.n, want_clouds, "kicp_register_staged_sensors",
                     voxel_map.ctx if f32_clouds else None)


def _segment_table(segments, what):
    """an (n, 16) float64 table of kicp_deskew_segment rows (t_begin, t_end, motion7, to_end7), 1 <= n <= KICP_MAX_DESKEW_SEGMENTS"""
    t = np.ascontiguousarray(segments, dtype=np.float64)
    if t.ndim != 2 or t.shape[1] != 16:
        raise ValueError("%s: an (n, 16) array of segments (t_begin, t_end, motion7, to_end7)" % what)
    if not 1 <= len(t) <= _capi.KICP_MAX_DESKEW_SEGMENTS:
        raise ValueError("%s: 1 to %d segments" % (what, _capi.KICP_MAX_DESKEW_SEGMENTS))
    return t


def RegisterStagedFrameSegments(voxel_map, staged, segments, lidar_to_base, last_pose, relative_odometry, tau, *, max_range=100.0,
                                min_range=0.0, deskew=True, voxel_size=1.0, max_num_iterations=10, convergence_criterion=0.001,
                                use_adaptive_odometry_regularization=True, fixed_regularization=0.0, want_clouds=True, f32_clouds=False):
    """kicp_register_staged_frame_segments: RegisterStagedFrame with the staged frame de-skewed along `segments` instead of one motion.
    `segments` is an (n, 16) array of kicp_deskew_segment rows (t_begin, t_end, motion7, to_end7) on the staged frame's clock, as
    deskew_segments builds them from odometry samples; relative_odometry keeps its role in the motion model and the threshold.  One
    segment [T0, T1] with the deskew motion and an identity to_end gives exactly what RegisterStagedFrame gives."""
    table = _segment_table(segments, "segments")
    fp = _frame_params(max_range, min_range, deskew, voxel_size, max_num_iterations, convergence_criterion,
                       use_adaptive_odometry_regularization, fixed_regularization)
    if f32_clouds:
        fp.stage_clouds = _capi.KICP_STAGE_F32
    args = (voxel_map.h, len(table), dp(table), dp(as_pose(lidar_to_base)), dp(as_pose(last_pose)), dp(as_pose(relative_odometry)),
            float(tau), C.byref(fp))
    return _register(lib().kicp_register_staged_frame_segments, args, staged.n, want_clouds, "kicp_register_staged_frame_segments",
                     voxel_map.ctx if f32_clouds else None)


def RegisterStagedSensorsSegments(voxel_map, staged, segments, lidar_to_bases, last_pose, relative_odometry, tau, *, max_range=100.0,
                                  min_range=0.0, deskew=True, voxel_size=1.0, max_num_iterations=10, convergence_criterion=0.001,
                                  use_adaptive_odometry_regularization=True, fixed_regularization=0.0, want_clouds=True, f32_clouds=False):
    """kicp_register_staged_sensors_segments: RegisterStagedSensors with sensor i de-skewed along segments[i] (an (n_i, 16) table as
    RegisterStagedFrameSegments takes it) instead of one motion."""
    k = getattr(staged, "k", 1)
    tables = [_segment_table(t, "segments[%d]" % i) for i, t in enumerate(segments)]
    l2bs = np.ascontiguousarray([as_pose(p) for p in lidar_to_bases], dtype=np.float64).reshape(-1, 7)
    if len(tables) != k or len(l2bs) != k:
        raise ValueError("one segment table and one lidar_to_base per staged sensor (%d)" % k)
    counts = np.array([len(t) for t in tables], dtype=np.int32)
    ptrs = (C.c_void_p * k)(*[t.ctypes.data for t in tables])
    fp = _frame_params(max_range, min_range, deskew, voxel_size, max_num_iterations, convergence_criterion,
                       use_adaptive_odometry_regularization, fixed_regularization)
    if f32_clouds:
        fp.stage_clouds = _capi.KICP_STAGE_F32
    args = (voxel_map.h, k, counts.ctypes.data, ptrs, dp(l2bs), dp(as_pose(last_pose)), dp(as_pose(relative_odometry)), float(tau),
            C.byref(fp))
    out = _register(lib().kicp_register_staged_sensors_segments, args, staged.n, want_clouds, "kicp_register_staged_sensors_segments",
                    voxel_map.ctx if f32_clouds else None)
    del tables
    return out


def shard_range(n, nranks, rank):
    """Contiguous index range [lo, hi) of rank `rank` out of `nranks` (SURVEY.md §8(e))."""
    return n * rank // nranks, n * (rank + 1) // nranks
