"""kicp_register_frame — KinematicICP::RegisterFrame (pipeline/KinematicICP.cpp:48-85) as one device-resident call —
against the CPU oracle stage by stage: Preprocess + base transform, both VoxelDownsamples, ComputeRobotMotion, map Update."""
import numpy as np
import pytest

import scenes as S
from test_gpu_parity import TOL_R, TOL_T, gpu_map_from_oracle, sorted_voxels

pytestmark = pytest.mark.gpu


def _oracle_frame(ko, w, om, frame, stamps, deskew_motion, l2b, deskew):
    pre = ko.preprocess(frame, stamps if deskew else np.zeros(0), deskew_motion, 100.0, 0.5, deskew)
    in_base = ko.se3_transform(l2b, pre)
    fd = ko.voxel_downsample(in_base, 0.5 * w.voxel_size)
    src = ko.voxel_downsample(fd, 1.5 * w.voxel_size)
    pose, stats = om.register(src, w.last_pose, w.rel_odom, w.tau)
    return in_base, fd, src, pose, stats


@pytest.mark.parametrize("frame_sync", [0, 1])  # 0: ONE host synchronisation per frame (default); 1: counts read back mid-frame
@pytest.mark.parametrize("deskew", [False, True])
def test_register_frame_matches_oracle_stages(oracle, gpu_ctx, workload, deskew, frame_sync):
    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(2)
    gpu_ctx.set_option("frame_sync", frame_sync)
    l2b = ko.se3_exp([0.2, -0.1, 0.3, 0.0, 0.0, 0.05])
    # the workload scan is in the base frame at true_pose: move it to the lidar frame, and add out-of-range clutter
    frame = ko.se3_transform(ko.se3_inverse(l2b), w.scan)
    frame = np.concatenate([frame, frame[:500] * 0.001, frame[:500] * 40.0])
    stamps = np.linspace(5.0, 5.1, len(frame))
    deskew_motion = ko.se3_compose(ko.se3_compose(ko.se3_inverse(l2b), w.rel_odom), l2b) if deskew else ko.IDENTITY
    om = ko.OracleMap(w.voxel_size, w.max_range, w.max_points_per_voxel)
    keys, counts, pts = w.map.export_voxels()
    om.add_points(pts)  # private copy of the workload map (voxel-grouped insertion keeps it identical)
    gm = gpu_map_from_oracle(kb, gpu_ctx, om)
    in_base, fd, src, opose, ostats = _oracle_frame(ko, w, om, frame, stamps, deskew_motion, l2b, deskew)
    try:
        pose, g_frame, g_src, res = kb.RegisterFrame(gm, frame, stamps, deskew_motion, l2b, w.last_pose, w.rel_odom, w.tau, max_range=100.0,
                                                     min_range=0.5, deskew=deskew, voxel_size=w.voxel_size)
        # the same frame against a fresh copy of the same map: this call plans its registration (grid, staging copy) from the first
        # one's survivor count instead of the worst case, and must land on the same pose
        gm2 = gpu_map_from_oracle(kb, gpu_ctx, om)
        pose2, _, g_src2, res2 = kb.RegisterFrame(gm2, frame, stamps, deskew_motion, l2b, w.last_pose, w.rel_odom, w.tau, max_range=100.0,
                                                  min_range=0.5, deskew=deskew, voxel_size=w.voxel_size)
    finally:
        gpu_ctx.set_option("frame_sync", 0)
    assert res.status == 0 and res.iterations == ostats.iterations
    d2 = ko.pose_delta(pose2, pose)
    assert res2.status == 0 and res2.iterations == res.iterations and d2[0] < 1e-12 and d2[1] < 1e-12 and np.array_equal(g_src2, g_src)
    if deskew:  # sin/cos of the de-skew differ in the last bits between device and glibc
        assert g_frame.shape == in_base.shape and np.abs(g_frame - in_base).max() < 1e-12
        assert g_src.shape == src.shape and np.abs(g_src - src).max() < 1e-12
    else:
        assert np.array_equal(g_frame, in_base) and np.array_equal(g_src, src)
    dt, dr = ko.pose_delta(pose, opose)
    assert dt < TOL_T and dr < TOL_R, (dt, dr)
    # the map received frame_downsample at the new pose and evicted far voxels: replay that on the oracle with the device's pose
    om.update_pose(fd, pose)
    assert gm.num_points() == om.num_points() and gm.num_voxels() == om.num_voxels()
    if not deskew:
        k1, c1, p1 = sorted_voxels(*gm.export_voxels())
        k0, c0, p0 = sorted_voxels(*om.export_voxels())
        assert np.array_equal(k1, k0) and np.array_equal(c1, c0) and np.array_equal(p1, p0)


def test_register_frame_float32_and_pointcloud2_layouts(oracle, gpu_ctx, workload):
    """float32 ingest (RosUtils.cpp:30-39 widens float32 fields to double): packed float32, a 16-byte x,y,z,intensity record and
    an unaligned record all give exactly the result of the widened float64 frame."""
    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(1)
    f32 = w.scan.astype(np.float32)
    wide = f32.astype(np.float64)
    ident = ko.IDENTITY
    args = (np.zeros(0), ident, ident, w.last_pose, w.rel_odom, w.tau)
    kw = dict(max_range=100.0, min_range=0.0, deskew=False, voxel_size=w.voxel_size)
    outs = []
    for variant in ("f64", "f32", "pc2", "unaligned"):
        gm = gpu_map_from_oracle(kb, gpu_ctx, w.map)
        if variant == "f64":
            r = kb.RegisterFrame(gm, wide, *args, **kw)
        elif variant == "f32":
            r = kb.RegisterFrame(gm, f32, *args, **kw)
        elif variant == "pc2":
            rec = np.zeros(len(f32), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("intensity", "<f4")])
            rec["x"], rec["y"], rec["z"], rec["intensity"] = f32[:, 0], f32[:, 1], f32[:, 2], 7.0
            r = kb.RegisterFrame(gm, rec, *args, point_step=16, offsets=(0, 4, 8), **kw)
        else:
            rec = np.zeros(len(f32), dtype=np.dtype({"names": ["tag", "z", "x", "y"], "formats": ["u1", "<f4", "<f4", "<f4"],
                                                      "offsets": [0, 1, 5, 9], "itemsize": 15}))
            rec["x"], rec["y"], rec["z"], rec["tag"] = f32[:, 0], f32[:, 1], f32[:, 2], 255
            r = kb.RegisterFrame(gm, rec, *args, point_step=15, offsets=(5, 9, 1), **kw)
        outs.append((r, sorted_voxels(*gm.export_voxels())))
    (p0, f0, s0, _), m0 = outs[0]
    assert np.array_equal(f0, wide)  # no filter, identity transform: the preprocessed frame is the widened input
    for (p, f, s, _), m in outs[1:]:
        assert np.array_equal(p, p0) and np.array_equal(f, f0) and np.array_equal(s, s0)
        assert all(np.array_equal(a, b) for a, b in zip(m, m0))


def test_register_frame_edge_cases(oracle, gpu_ctx, workload):
    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(1)
    ident = ko.IDENTITY
    # first frame of a drive: empty map -> the pose is the prediction (Registration.cpp:157) and the map gets the frame
    gm = kb.VoxelHashMap(gpu_ctx, w.voxel_size, w.max_range, w.max_points_per_voxel)
    pose, frame, src, res = kb.RegisterFrame(gm, w.scan, np.zeros(0), ident, ident, w.last_pose, w.rel_odom, w.tau, voxel_size=w.voxel_size)
    dt, dr = ko.pose_delta(pose, w.prior)
    assert dt < 1e-12 and dr < 1e-12 and res.iterations == 0
    om = ko.OracleMap(w.voxel_size, w.max_range, w.max_points_per_voxel)
    om.update_pose(ko.voxel_downsample(w.scan, 0.5 * w.voxel_size), pose)
    assert gm.num_points() == om.num_points() > 0
    # empty frame against a non-empty map: zero correspondences -> NaN pose like the reference, flagged, map untouched
    before = gm.num_points()
    pose, frame, src, res = kb.RegisterFrame(gm, np.zeros((0, 3)), np.zeros(0), ident, ident, w.last_pose, w.rel_odom, w.tau,
                                             voxel_size=w.voxel_size)
    assert len(frame) == 0 and len(src) == 0 and np.isnan(pose).any() and res.status == kb.KICP_WARN_NO_CORRESPONDENCES
    assert gm.num_points() == before
    # every point outside the range gate: same
    pose, frame, src, res = kb.RegisterFrame(gm, w.scan[:100] * 1e-4, np.zeros(0), ident, ident, w.last_pose, w.rel_odom, w.tau,
                                             min_range=0.5, voxel_size=w.voxel_size)
    assert len(frame) == 0 and res.status == kb.KICP_WARN_NO_CORRESPONDENCES and gm.num_points() == before
    # without cloud downloads
    gm2 = gpu_map_from_oracle(kb, gpu_ctx, w.map)
    gm3 = gpu_map_from_oracle(kb, gpu_ctx, w.map)
    a = kb.RegisterFrame(gm2, w.scan, np.zeros(0), ident, ident, w.last_pose, w.rel_odom, w.tau, voxel_size=w.voxel_size)
    b = kb.RegisterFrame(gm3, w.scan, np.zeros(0), ident, ident, w.last_pose, w.rel_odom, w.tau, voxel_size=w.voxel_size, want_clouds=False)
    assert np.array_equal(a[0], b[0]) and b[1] == len(a[1]) and b[2] == len(a[2])


def _frame_capi(kb, gm, frame, cap_frame, cap_source, voxel_size):
    """kicp_register_frame with caller buffers of the given capacities (the Python wrapper always passes enough)."""
    import ctypes as C
    from kinematic_icp_b200 import _capi
    from kinematic_icp_b200._capi import FrameInput, FrameParams, RegResult, dp
    inp = FrameInput()
    inp.data, inp.n, inp.dtype, inp.point_step = frame.ctypes.data, len(frame), _capi.KICP_DTYPE_F64, 0
    fp = FrameParams()
    fp.max_range, fp.min_range, fp.deskew, fp.voxel_size = 100.0, 0.5, 0, voxel_size
    fp.reg.max_num_iterations, fp.reg.use_adaptive_odometry_regularization, fp.reg.convergence_criterion = 10, 1, 1e-3
    ident = np.array([0, 0, 0, 1.0, 0, 0, 0])
    out_pose, out_f, out_s = np.empty(7), np.empty((max(cap_frame, 1), 3)), np.empty((max(cap_source, 1), 3))
    nf, ns, res = C.c_int64(), C.c_int64(), RegResult()
    st = _capi.lib().kicp_register_frame(gm.h, C.byref(inp), dp(ident), dp(ident), dp(ident), dp(ident), 1.0, C.byref(fp), dp(out_pose),
                                         dp(out_f), cap_frame, C.byref(nf), dp(out_s), cap_source, C.byref(ns), C.byref(res))
    return st, nf.value, ns.value


def test_register_frame_drive(oracle, monkeypatch):
    """Twelve frames through kicp_register_frame on a context of their own and a map that starts at its smallest slab, each checked
    against the oracle stage by stage: the preprocessed frame and the source bit for bit (1e-12 with de-skew), the pose to
    1e-6 m / 1e-7 rad, the map bit for bit after the device's pose is replayed on the oracle's.  The drive holds a tiny frame followed
    by one whose source exceeds max(2 x previous, 32 768) (the rest-of-source fetch, and a registration planned from a far smaller
    frame), an empty frame and one with every point outside the range gate (NaN pose, flagged, map untouched), a frame that grows the
    front end's scratch, growth of the map's slab inside the asynchronous update, de-skew, float32 and PointCloud2 layouts, and
    frame_sync 0 and 1.  Then a caller buffer too small for the survivors: KICP_ERR_CAPACITY, the map unchanged, and
    kicp_frame_clouds still holding the last frame's clouds."""
    import ctypes as C

    import kinematic_icp_b200 as kb
    from kinematic_icp_b200 import _capi
    ko = oracle
    monkeypatch.setenv("KICP_MAP_VOXELS", "16384")
    vs, md, cap, tau = 1.0, 40.0, 20, 1.0
    rng = np.random.default_rng(2026)
    world = np.c_[rng.uniform(-45.0, 85.0, 420_000), rng.uniform(-50.0, 50.0, 420_000), rng.uniform(-3.0, 12.0, 420_000)]
    world = np.round(world * 4096.0) / 4096.0
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, vs, md, cap)
    om = ko.OracleMap(vs, md, cap)
    l2b = ko.se3_exp([0.1, 0.0, 0.2, 0.0, 0.0, 0.02])
    step = ko.se3_exp([2.5, 0.1, 0.0, 0.0, 0.0, 0.01])
    true_pose = ko.IDENTITY.copy()
    last = ko.IDENTITY.copy()
    # (kind, frame_sync): how each frame is built and handed over
    plan = [("tiny", 0), ("big", 0), ("empty", 0), ("gated", 0), ("sub", 1), ("deskew", 0), ("f32", 0), ("pc2", 0), ("huge", 0), ("sub", 0),
            ("deskew", 1), ("sub", 0)]
    prev_source, last_clouds = 0, None
    try:
        for k, (kind, sync) in enumerate(plan):
            odom = step if k else ko.IDENTITY.copy()
            true_pose = ko.se3_compose(true_pose, odom)
            lidar = ko.se3_transform(ko.se3_inverse(ko.se3_compose(true_pose, l2b)), world)  # the world in this frame's lidar frame
            r = np.sqrt((lidar * lidar).sum(1))
            lidar = lidar[(r < 100.0)]
            stamps = np.zeros(0)
            deskew_motion = ko.IDENTITY
            if kind == "tiny":
                frame = lidar[:150]
            elif kind == "big":
                frame = lidar
            elif kind == "empty":
                frame = np.zeros((0, 3))
            elif kind == "gated":
                frame = lidar[:3000] * 1e-4
            elif kind == "huge":  # more points than any frame before: the scratch grows
                frame = np.concatenate([lidar, lidar[::2] + 0.01])
            else:
                frame = lidar[k % 3::3]
            if kind in ("f32", "pc2"):
                frame = frame.astype(np.float32)
            wide = frame.astype(np.float64)
            if kind == "deskew":
                stamps = np.linspace(7.0, 7.1, len(frame))
                deskew_motion = ko.se3_compose(ko.se3_compose(ko.se3_inverse(l2b), odom), l2b)
            ctx.set_option("frame_sync", sync)
            if kind == "pc2":
                rec = np.zeros(len(frame), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("i", "<f4")])
                rec["x"], rec["y"], rec["z"], rec["i"] = frame[:, 0], frame[:, 1], frame[:, 2], 3.0
                arg, extra = rec, dict(point_step=16, offsets=(0, 4, 8))
            else:
                arg, extra = frame, {}
            before = sorted_voxels(*gm.export_voxels())
            pose, g_frame, g_src, res = kb.RegisterFrame(gm, arg, stamps, deskew_motion, l2b, last, odom, tau, max_range=100.0, min_range=0.5,
                                                         deskew=kind == "deskew", voxel_size=vs, **extra)
            # the oracle, stage by stage
            pre = ko.preprocess(wide, stamps, deskew_motion, 100.0, 0.5, kind == "deskew")
            in_base = ko.se3_transform(l2b, pre) if len(pre) else np.zeros((0, 3))
            fd = ko.voxel_downsample(in_base, 0.5 * vs) if len(in_base) else np.zeros((0, 3))
            src = ko.voxel_downsample(fd, 1.5 * vs) if len(fd) else np.zeros((0, 3))
            assert g_frame.shape == in_base.shape and g_src.shape == src.shape, kind
            if kind == "deskew":
                assert np.abs(g_frame - in_base).max() < 1e-12 and np.abs(g_src - src).max() < 1e-12
            else:
                assert S.same_bits(g_frame, in_base) and S.same_bits(g_src, src), kind
            if kind == "big":
                assert len(src) > max(2 * prev_source, 32768), (len(src), prev_source)
            prev_source = len(src)
            if len(src) == 0:  # nothing to register: the reference's NaN pose, flagged, the map untouched
                assert np.isnan(pose).any() and res.status == kb.KICP_WARN_NO_CORRESPONDENCES, kind
                after = sorted_voxels(*gm.export_voxels())
                assert all(np.array_equal(a, b) for a, b in zip(before, after))
                continue
            # the oracle registers the device's source (bit-identical, or within 1e-12 under de-skew)
            opose, ost = om.register(g_src, last, odom, tau)
            assert res.status == 0 and res.iterations == ost.iterations, kind
            dt, dr = ko.pose_delta(pose, opose)
            assert dt < TOL_T and dr < TOL_R, (kind, dt, dr)
            # the map received the device's frame_downsample at the device's pose
            om.update_pose(ko.voxel_downsample(g_frame, 0.5 * vs), pose)
            k1, c1, p1 = sorted_voxels(*gm.export_voxels())
            k0, c0, p0 = sorted_voxels(*om.export_voxels())
            assert np.array_equal(k1, k0) and np.array_equal(c1, c0) and S.same_bits(p1, p0), kind
            last, last_clouds = pose, (g_frame, g_src)
        assert gm.num_voxels() > 16384  # the slab grew during the drive
        # a caller buffer too small for the survivors: KICP_ERR_CAPACITY before the map changes
        ctx.set_option("frame_sync", 0)
        before = sorted_voxels(*gm.export_voxels())
        frame = np.ascontiguousarray(ko.se3_transform(ko.se3_inverse(ko.se3_compose(true_pose, l2b)), world[::50]))
        st, nf, ns = _frame_capi(kb, gm, frame, 10, len(frame), vs)
        assert st == _capi.KICP_ERR_CAPACITY and nf > 10
        after = sorted_voxels(*gm.export_voxels())
        assert all(S.same_bits(a, b) if a.dtype == np.float64 else np.array_equal(a, b) for a, b in zip(before, after))
        fp_, fs_ = C.POINTER(C.c_double)(), C.POINTER(C.c_double)()
        n_f, n_s = C.c_int64(), C.c_int64()
        assert _capi.lib().kicp_frame_clouds(ctx.h, C.byref(fp_), C.byref(n_f), C.byref(fs_), C.byref(n_s)) == 0
        got_f = np.ctypeslib.as_array(fp_, shape=(n_f.value * 3,)).reshape(-1, 3).copy()
        got_s = np.ctypeslib.as_array(fs_, shape=(n_s.value * 3,)).reshape(-1, 3).copy()
        assert S.same_bits(got_f, last_clouds[0]) and S.same_bits(got_s, last_clouds[1])
    finally:
        gm.close()
        ctx.close()
