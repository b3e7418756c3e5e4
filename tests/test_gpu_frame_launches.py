"""The frame path's launch sequence, call by call: kicp_register_frame, kicp_frame_stage + kicp_register_staged_frame and
kicp_frame_stage_laser_scan + kicp_register_staged_frame, in both synchronisation orders (option frame_sync 0: one host
synchronisation per frame; 1: the survivor counts read back mid-frame) and with stage_clouds 0 / 1 / 2 / 3.  Every call's
ctx.launch_count difference is pinned, and so are the clouds it stages (kicp_frame_clouds, kicp_frame_clouds_f32).

Each map is warmed up with its own frame first, and every point lies well inside max_distance, so the pinned frames neither grow the
map's slab or hash table nor evict a voxel (an eviction would add a compaction to the read-back order's map update)."""
import ctypes as C

import numpy as np
import pytest

import scenes as S
from test_gpu_publish import _clouds, _frame_params, bits32

pytestmark = pytest.mark.gpu

IDENT = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
MOTION = np.array([0.0, 0.0, np.sin(0.005), np.cos(0.005), 0.05, 0.0, 0.0])  # de-skew motion of a sweep
VS = 1.0
# launches of one frame on a non-empty map
FRONT = 1 + 3 + 3  # k_preprocess_select; two down-samples of k_ds_clear + k_ds_insert + k_ds_select each
REG = 1  # k_register, all IRLS passes in one persistent launch
MAP = {0: 6,  # k_add_find_or_create, k_add_commit, k_mark_far, k_exclusive_sum, k_compact_blocks, k_table_rebuild
       1: 3}  # k_add_find_or_create, k_add_commit, k_mark_far (nothing evicted, so nothing compacted)


def _world(n=40000, seed=7):
    rng = np.random.default_rng(seed)
    pts = np.c_[rng.uniform(-30.0, 30.0, n), rng.uniform(-30.0, 30.0, n), rng.uniform(-2.0, 6.0, n)]
    return np.round(pts * 4096.0) / 4096.0 + 0.0  # exact in float32 too; no -0.0


def _records(xyz, with_time):
    """20-byte PointCloud2-style records: float32 x, y, z, intensity, then (with_time) uint32 nanoseconds since the sweep start"""
    dt = np.dtype({"names": ["x", "y", "z", "i", "t"], "formats": ["<f4", "<f4", "<f4", "<f4", "<u4"], "offsets": [0, 4, 8, 12, 16],
                   "itemsize": 20})
    rec = np.zeros(len(xyz), dtype=dt)
    rec["x"], rec["y"], rec["z"], rec["i"] = xyz[:, 0], xyz[:, 1], xyz[:, 2], 1.0
    if with_time:
        rec["t"] = np.round(np.linspace(0.0, 1e8, len(xyz))).astype(np.uint32)
    return np.frombuffer(rec.tobytes(), dtype=np.uint8)


def _register(ctx, gm, inp, stage, deskew, cap=None):
    """kicp_register_frame (inp: a kicp_frame_input) or kicp_register_staged_frame (inp None), with caller buffers of `cap` points or
    none: (status, launches, (n_frame, n_source), staged clouds)"""
    from kinematic_icp_b200 import _capi
    from kinematic_icp_b200._capi import RegResult, dp
    L = _capi.lib()
    fp = _frame_params(stage, deskew, VS, min_range=0.0)
    out_pose, res, nf, ns = np.empty(7), RegResult(), C.c_int64(), C.c_int64()
    bufs = [np.empty((max(cap, 1), 3)) for _ in range(2)] if cap is not None else None
    tail = (dp(out_pose), dp(bufs[0]) if bufs else None, cap or 0, C.byref(nf), dp(bufs[1]) if bufs else None, cap or 0, C.byref(ns),
            C.byref(res))
    poses = (dp(MOTION if deskew else IDENT), dp(IDENT), dp(IDENT), dp(IDENT))
    l0 = ctx.launch_count
    if inp is None:
        st = L.kicp_register_staged_frame(gm.h, *poses, 1.0, C.byref(fp), *tail)
    else:
        st = L.kicp_register_frame(gm.h, C.byref(inp), *poses, 1.0, C.byref(fp), *tail)
    return st, ctx.launch_count - l0, (nf.value, ns.value), _clouds(ctx)


class _Kind:
    """one way a frame reaches the registration: stage() (launches of the staging call, 0 when there is none), then register()"""

    def __init__(self, kind, world):
        import kinematic_icp_b200 as kb
        self.kind, self.kb = kind, kb
        self.deskew = kind in ("deskew", "staged_time", "laser")
        self.extra = 0  # launches of kicp_register_frame before its front end
        self.inp = None
        if kind == "f64":
            self.inp, self.keep, _ = kb._frame_input(world, np.zeros(0), 0, (0, 0, 0))
        elif kind == "f32_strided":
            self.inp, self.keep, _ = kb._frame_input(_records(world, False), np.zeros(0), 20, (0, 4, 8))
            self.extra = 1  # k_ingest
        elif kind == "deskew":
            self.inp, self.keep, _ = kb._frame_input(world, np.linspace(0.0, 0.1, len(world)), 0, (0, 0, 0))
            self.extra = 1  # k_stamp_minmax of the host stamps
        elif kind == "laser":
            beams = 1440
            self.ranges = (8.0 + 4.0 * np.sin(np.arange(beams) * 0.05)).astype(np.float32)
        self.world = world

    def stage(self, ctx):
        """launches of the staging call"""
        kb = self.kb
        l0 = ctx.launch_count
        if self.kind == "staged_plain":  # packed float64, no time field: one copy, no launch
            sf = kb.StageFrame(ctx, self.world)
            assert sf.n == len(self.world) and sf.n_stamps == 0
        elif self.kind == "staged_time":  # k_ingest_stamped + k_stamp_minmax
            sf = kb.StageFrame(ctx, _records(self.world, True), point_step=20, offsets=(0, 4, 8), stamp_datatype=6, stamp_offset=16)
            assert sf.n == sf.n_stamps == len(self.world)
        elif self.kind == "laser":  # k_laser_project_select + k_stamp_minmax
            sf = kb.StageLaserScan(ctx, self.ranges, angle_min=-np.pi, angle_max=np.pi - 2 * np.pi / len(self.ranges),
                                   angle_increment=2 * np.pi / len(self.ranges), time_increment=1e-5, range_min=0.1, range_max=30.0)
            assert sf.n == len(self.ranges)
        return ctx.launch_count - l0

    def register(self, ctx, gm, stage, cap=None):
        return _register(ctx, gm, self.inp, stage, self.deskew, cap)


STAGE_LAUNCHES = {"f64": 0, "f32_strided": 0, "deskew": 0, "staged_plain": 0, "staged_time": 2, "laser": 2}


@pytest.mark.parametrize("kind", ["f64", "f32_strided", "deskew", "staged_plain", "staged_time", "laser"])
def test_frame_launches_and_staged_clouds(kind):
    import kinematic_icp_b200 as kb
    world = _world()
    k = _Kind(kind, world)
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, VS, 100.0, 20)
    try:
        for _ in range(3):  # warm-up: the map holds the frame's voxels, its table is sized for them
            k.stage(ctx)
            st, _, _, _ = k.register(ctx, gm, 0)
            assert st == 0
        ref = None
        for sync in (0, 1):
            ctx.set_option("frame_sync", sync)
            for stage in (3, 0, 1, 2):
                assert k.stage(ctx) == STAGE_LAUNCHES[kind], (sync, stage)
                st, launches, (nf, ns), (df, ds, ff, fs) = k.register(ctx, gm, stage)
                assert st == 0, (sync, stage, st)
                assert launches == k.extra + FRONT + (1 if stage & 2 else 0) + REG + MAP[sync], (sync, stage, launches)
                if ref is None:  # stage_clouds 3, default order: both encodings
                    ref = (df, ds)
                    assert len(df) == nf > 0 and len(ds) == ns > 0
                assert (nf, ns) == (len(ref[0]), len(ref[1]))
                if stage & 1:
                    assert S.same_bits(df, ref[0]) and S.same_bits(ds, ref[1]), (sync, stage)
                else:
                    assert len(df) == len(ds) == 0
                if stage & 2:
                    assert np.array_equal(bits32(ff), bits32(ref[0])) and np.array_equal(bits32(fs), bits32(ref[1])), (sync, stage)
                else:
                    assert len(ff) == len(fs) == 0
            # caller buffers (the doubles are staged whatever stage_clouds says): both orders as above
            assert k.stage(ctx) == STAGE_LAUNCHES[kind]
            st, launches, _, (df, ds, _, _) = k.register(ctx, gm, 0, cap=len(world))
            assert st == 0 and launches == k.extra + FRONT + REG + MAP[sync], (sync, launches)
            assert S.same_bits(df, ref[0]) and S.same_bits(ds, ref[1])
        ctx.set_option("frame_sync", 0)
        if kind in ("f64", "f32_strided"):  # identity lidar_to_base, no range gate in reach: the frame is the input, widened
            assert np.array_equal(ref[0], world)
            assert S.same_bits(ref[1], kb.VoxelDownsample(ctx, kb.VoxelDownsample(ctx, world, 0.5 * VS), 1.5 * VS))
    finally:
        gm.close()
        ctx.close()


def test_frame_launches_empty_frame_and_capacity_error():
    """An empty frame launches the registration alone (no correspondences: the map is not updated).  A caller buffer too small for
    the survivors takes the read-back order and returns KICP_ERR_CAPACITY after the front end, before the registration: the previous
    frame's clouds stay staged."""
    import kinematic_icp_b200 as kb
    from kinematic_icp_b200 import _capi
    world = _world()
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, VS, 100.0, 20)
    try:
        inp, keep, _ = kb._frame_input(world, np.zeros(0), 0, (0, 0, 0))
        for _ in range(3):
            assert _register(ctx, gm, inp, 0, False)[0] == 0
        st, launches, counts, (df, ds, ff, fs) = _register(ctx, gm, inp, 3, False)
        assert st == 0 and launches == FRONT + 1 + REG + MAP[0]
        before = gm.num_points()
        for sync in (0, 1):
            ctx.set_option("frame_sync", sync)
            e_inp, e_keep, _ = kb._frame_input(np.zeros((0, 3)), np.zeros(0), 0, (0, 0, 0))
            st, launches, (nf, ns), clouds = _register(ctx, gm, e_inp, 3, False)
            assert st == _capi.KICP_WARN_NO_CORRESPONDENCES and launches == REG and nf == ns == 0
            assert all(len(c) == 0 for c in clouds) and gm.num_points() == before
            assert _register(ctx, gm, inp, 3, False)[:2] == (0, FRONT + 1 + REG + MAP[sync])
            st, launches, (nf, ns), clouds = _register(ctx, gm, inp, 3, False, cap=10)
            assert st == _capi.KICP_ERR_CAPACITY and launches == FRONT + 1 and (nf, ns) == counts
            assert S.same_bits(clouds[0], df) and S.same_bits(clouds[1], ds)
            assert np.array_equal(bits32(clouds[2]), bits32(ff)) and np.array_equal(bits32(clouds[3]), bits32(fs))
        del keep, e_keep
    finally:
        ctx.set_option("frame_sync", 0)
        gm.close()
        ctx.close()
