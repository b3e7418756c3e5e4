"""The pose search on the GPU (kicp_map_pose_search, kicp_map_pose_search_device through VoxelHashMap.PoseSearch) against the oracle's
restatement (tests/pose_search_oracle.py): an exhaustive single-level grid hypothesis by hypothesis, also against Correspondences at
each pose; a multi-level search on cfg2; recovery of a known planar perturbation of cfg2's true pose; host, device float64 and strided
float32 device inputs; repeated calls; no side effect on the map; an empty map and n = 0."""
import math

import numpy as np
import pytest

import pose_search_oracle as PO

pytestmark = pytest.mark.gpu


def _map(kb, ctx, w):
    gm = kb.VoxelHashMap(ctx, w.voxel_size, w.max_range, w.max_points_per_voxel)
    gm.load_voxels(*w.map.export_voxels())
    return gm


def _src(w, n):
    return np.ascontiguousarray(w.scan[:: max(1, len(w.scan) // n)][:n], dtype=np.float64)


def test_exhaustive_grid(oracle, workload):
    """levels = 1 and keep = every hypothesis (4 x 4 x 4 = 64 at most: a 3 x 3 x 3 grid here plus nothing else): each one the oracle's
    (count exactly, sum_sq bit for bit in the kernel's order and 1e-12 of the plain sum, pose bits), and each one's count and sum the
    Correspondences report's at its pose"""
    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(2)
    ctx = kb.Context(0)
    gm = _map(kb, ctx, w)
    try:
        src = _src(w, 3000)
        prior = ko.se3_compose(w.true_pose, ko.planar_pose(0.05, -0.03, 0.01))
        he, st = (0.3, 0.3, 0.02), (0.3, 0.3, 0.02)
        res = PO.search(ko, w.map, src, prior, w.tau, he, st, 1, 27)
        hyps, n_scored = gm.PoseSearch(src, prior, w.tau, he, st, levels=1, keep=27)
        assert n_scored == 27 == res["n_scored"]
        PO.check_hypotheses(hyps, res, prior, len(src))
        for h in hyps:
            *_, cs = gm.Correspondences(src, h.pose, w.tau)
            assert cs.n_inliers == h.n_inliers
            assert abs(cs.sum_sq - h.sum_sq) <= 1e-12 * abs(cs.sum_sq)
        assert hyps[0].n_inliers > hyps[-1].n_inliers
    finally:
        gm.close()
        ctx.close()


def test_multi_level_cfg2(oracle, workload):
    """three levels, keep 8, on cfg2: the output's lattice points, levels and counts equal the oracle search's; no near-tie in the
    oracle's plain sums, so a ranking difference could not be rounding"""
    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(2)
    ctx = kb.Context(0)
    gm = _map(kb, ctx, w)
    try:
        src = _src(w, 2000)
        prior = ko.se3_compose(w.true_pose, ko.planar_pose(0.21, 0.13, -0.03))
        he, st = (0.4, 0.4, 0.06), (0.2, 0.2, 0.03)
        res = PO.search(ko, w.map, src, prior, w.tau, he, st, 3, 8)
        assert not PO.near_tie(res)
        hyps, n_scored = gm.PoseSearch(src, prior, w.tau, he, st, levels=3, keep=8)
        assert n_scored == res["n_scored"]
        PO.check_hypotheses(hyps, res, prior, len(src))
    finally:
        gm.close()
        ctx.close()


def _planar_inverse(x, y, yaw):
    c, s = math.cos(-yaw), math.sin(-yaw)
    return np.array([-(c * x - s * y), -(s * x + c * y), -yaw])


def test_recovery_cfg2(oracle, workload):
    """a prior perturbed from cfg2's true pose by a known off-lattice (x, y, yaw): the best hypothesis's offset is within one finest
    step of the offset that undoes it, on each axis.  The gate is a few finest steps wide (0.15 m): with the registration's adaptive
    gate (0.97 m here) nearly every point is an inlier over much of the grid and the count no longer tells the offsets apart."""
    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(2)
    ctx = kb.Context(0)
    gm = _map(kb, ctx, w)
    try:
        src = _src(w, 1000)
        d = (0.37, -0.23, 0.041)
        prior = ko.se3_compose(w.true_pose, ko.planar_pose(*d))
        he, st, levels = (0.8, 0.8, 0.08), (0.2, 0.2, 0.04), 3
        hyps, _ = gm.PoseSearch(src, prior, 0.15, he, st, levels=levels, keep=8)
        fine = np.array(st) / 2 ** (levels - 1)
        err = np.abs(np.array(hyps[0].offset) - _planar_inverse(*d))
        assert (err <= fine).all(), (hyps[0].offset, _planar_inverse(*d), err)
    finally:
        gm.close()
        ctx.close()


def test_inputs_repeat_and_no_side_effects(oracle, workload):
    """host float64, device float64 and strided float32 device records give the same output (float32 points widened exactly);
    a repeated call the same bits; the map's export_voxels unchanged by a search"""
    import torch

    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(2)
    ctx = kb.Context(0)
    gm = _map(kb, ctx, w)
    try:
        src = _src(w, 1500).astype(np.float32).astype(np.float64)
        prior = ko.se3_compose(w.true_pose, ko.planar_pose(0.1, 0.0, 0.02))
        he, st = (0.3, 0.3, 0.04), (0.1, 0.1, 0.02)
        before = gm.export_voxels()
        a, na = gm.PoseSearch(src, prior, w.tau, he, st, levels=2, keep=6)
        b, nb = gm.PoseSearch(src, prior, w.tau, he, st, levels=2, keep=6)
        dev = torch.from_numpy(src).cuda()
        c, nc = gm.PoseSearch(dev, prior, w.tau, he, st, levels=2, keep=6)
        rec = torch.zeros((len(src), 5), dtype=torch.float32, device="cuda")
        rec[:, 1:4] = torch.from_numpy(src.astype(np.float32)).cuda()
        e, ne = gm.PoseSearch(rec, prior, w.tau, he, st, levels=2, keep=6, point_step=20, offsets=(4, 8, 12))
        res = PO.search(ko, w.map, src, prior, w.tau, he, st, 2, 6)
        assert na == nb == nc == ne == res["n_scored"]
        for got in (a, b, c, e):
            assert len(got) == len(a)
            for x, y in zip(got, a):
                assert np.array_equal(x.pose, y.pose) and x[1:] == y[1:]
        PO.check_hypotheses(a, res, prior, len(src))
        after = gm.export_voxels()
        assert all(np.array_equal(x, y) for x, y in zip(before, after))
    finally:
        gm.close()
        ctx.close()


def test_empty_map_and_n0(oracle):
    """an empty map and n = 0: every score (0, 0), the keep lattice points nearest the prior by the key"""
    import kinematic_icp_b200 as kb
    ko = oracle
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, 1.0, 100.0, 20)
    try:
        om = ko.OracleMap(1.0, 100.0, 20)
        pts = np.random.default_rng(3).uniform(-5, 5, (300, 3))
        prior = ko.planar_pose(1.0, 2.0, 0.3)
        for src in (pts, np.zeros((0, 3))):
            res = PO.search(ko, om, src, prior, 0.5, (0.2, 0.2, 0.1), (0.1, 0.1, 0.1), 2, 5)
            hyps, n = gm.PoseSearch(src, prior, 0.5, (0.2, 0.2, 0.1), (0.1, 0.1, 0.1), levels=2, keep=5)
            assert n == res["n_scored"]
            PO.check_hypotheses(hyps, res, prior, len(src))
            assert hyps[0].lattice == (0, 0, 0) and all(h.n_inliers == 0 for h in hyps)
    finally:
        gm.close()
        ctx.close()


def _pose_hooks():
    import ctypes as C
    import os
    from test_gpu_laserscan import _laser_hooks
    L, P, Q = _laser_hooks()
    H = C.CDLL(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "hooks", "_build",
                            "libkicp_pose_search_hooks.so"))
    H.kfps_map_create.restype = C.c_void_p
    H.kfps_map_create.argtypes = [C.c_double, C.c_double, C.c_uint]
    H.kfps_map_destroy.argtypes = [C.c_void_p]
    H.kfps_map_add_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    H.kfps_map_handle.restype = C.c_void_p
    H.kfps_map_handle.argtypes = [C.c_void_p]
    for f in (H.kfps_map_search_pose, H.kfps_pipeline_search_pose):
        f.restype = C.c_int32
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.POINTER(PO.Params), C.POINTER(PO.Hypothesis)]
    H.kfps_pipeline_assign_pose.argtypes = [C.c_void_p, C.c_void_p]
    H.kfps_pipeline_pose.argtypes = [C.c_void_p, C.c_void_p]
    return L, P, Q, H


def test_facade_search_pose_equals_c_call(oracle, workload):
    """kiss_icp::VoxelHashMap::SearchPose (tests/hooks/pose_search_hooks.cpp) == kicp_map_pose_search on the same map: every field bit
    for bit except the pose, which passes through Sophus (from_pose7 normalises the quaternion again) and agrees to 1e-15"""
    import ctypes as C

    from kinematic_icp_b200 import _capi
    ko = oracle
    w = workload(2)
    _, _, _, H = _pose_hooks()
    lib = _capi.lib()
    m = H.kfps_map_create(w.voxel_size, w.max_range, w.max_points_per_voxel)
    try:
        pts = np.ascontiguousarray(w.map.pointcloud(), dtype=np.float64)
        H.kfps_map_add_points(m, pts.ctypes.data, len(pts))
        src = _src(w, 1500)
        prior = np.ascontiguousarray(ko.se3_compose(w.true_pose, ko.planar_pose(0.12, -0.08, 0.02)))
        p = PO.params((0.3, 0.3, 0.04), (0.1, 0.1, 0.02), 0.3, 2, 6)
        a = (PO.Hypothesis * 6)()
        na = H.kfps_map_search_pose(m, src.ctypes.data, len(src), prior.ctypes.data, C.byref(p), a)
        b = (PO.Hypothesis * 6)()
        nb, ns = C.c_int32(), C.c_int64()
        _capi.check(lib.kicp_map_pose_search(C.c_void_p(H.kfps_map_handle(m)), _capi.dp(src), len(src), _capi.dp(prior),
                                             C.cast(C.byref(p), C.POINTER(_capi.PoseSearchParams)),
                                             C.cast(b, C.POINTER(_capi.PoseHypothesis)), 6, C.byref(nb), C.byref(ns)),
                    "kicp_map_pose_search")
        assert na == nb.value == 6
        for x, y in zip(a, b):
            assert np.abs(np.array(x.pose[:]) - np.array(y.pose[:])).max() <= 1e-15
            assert bytes(x)[C.sizeof(C.c_double) * 7:] == bytes(y)[C.sizeof(C.c_double) * 7:]
        assert b[0].n_inliers > 0
    finally:
        H.kfps_map_destroy(m)


def test_laser_scan_recovery_and_pose_assignment_keeps_the_map(oracle):
    """The 2D golden drive (tests/golden/pipeline_2d.npz) through kinematic_icp::pipeline::KinematicICP for 12 frames; then frame 12's
    LaserScan, projected into the base frame, searched on the pipeline's map (SearchPose on VoxelMap()) from the reference's pose of
    that frame perturbed by a known off-lattice (x, y, yaw): the best hypothesis is within one finest step of the offset that undoes
    it.  `pose() = hyps[0].pose` keeps the map (SetPose clears it), and frame 13 registered from there lands near the reference's pose."""
    import ctypes as C
    import os
    import sys

    import laser_projection as LP
    ko = oracle
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "tests", "golden"))
    import make_golden_2d as G
    z = np.load(os.path.join(root, "tests", "golden", "pipeline_2d.npz"))
    l2b, start, frames = G.unpack(z)
    l2b, start = np.ascontiguousarray(l2b, dtype=np.float64), np.ascontiguousarray(start, dtype=np.float64)
    L, P, Q, H = _pose_hooks()
    p = L.kfac_pipeline_create(100.0, 0.0, 1.0, 20, 1, 1.0, 10, 1e-3, 1, 1, 0.0, 0)
    K = 12
    try:
        L.kfac_pipeline_set_pose(p, start.ctypes.data)
        last = np.zeros(1)

        def register(k):
            ranges, kw, header, odom = frames[k]
            ranges = np.ascontiguousarray(ranges, dtype=np.float32)
            odom = np.ascontiguousarray(odom, dtype=np.float64)
            prm = np.array([kw[q] for q in G.PARAMS], dtype=np.float32)
            be, pose = np.zeros(2), np.zeros(7)
            assert Q.kfac_pipeline_stage_laser_scan(p, ranges.ctypes.data, len(ranges), prm.ctypes.data, header, last.ctypes.data,
                                                    be.ctypes.data) == 0
            return P.kfac_pipeline_register_staged(p, l2b.ctypes.data, odom.ctypes.data, pose.ctypes.data), pose

        for k in range(K):
            register(k)
        n_map = L.kfac_pipeline_num_map_points(p)
        assert n_map > 0
        ranges, kw, _, _ = frames[K]
        scan = LP.LaserProjector().project(ranges, **kw)["points"]
        src = np.ascontiguousarray(ko.se3_transform(l2b, np.asarray(scan, dtype=np.float64)))
        truth = z["plain_poses"][K]
        d = (0.23, -0.17, 0.031)
        prior = np.ascontiguousarray(ko.se3_compose(truth, ko.planar_pose(*d)))
        levels, st = 3, (0.2, 0.2, 0.04)
        prm = PO.params((0.6, 0.6, 0.08), st, 0.15, levels, 8)
        hyps = (PO.Hypothesis * 8)()
        n = H.kfps_pipeline_search_pose(p, src.ctypes.data, len(src), prior.ctypes.data, C.byref(prm), hyps)
        assert n == 8
        fine = np.array(st) / 2 ** (levels - 1)
        err = np.abs(np.array(hyps[0].offset[:]) - _planar_inverse(*d))
        assert (err <= fine).all(), (list(hyps[0].offset), _planar_inverse(*d), err)
        assert L.kfac_pipeline_num_map_points(p) == n_map  # the search leaves the map alone
        best = np.ascontiguousarray(hyps[0].pose[:])
        H.kfps_pipeline_assign_pose(p, best.ctypes.data)
        got = np.zeros(7)
        H.kfps_pipeline_pose(p, got.ctypes.data)
        assert np.abs(got - best).max() <= 1e-15
        assert L.kfac_pipeline_num_map_points(p) == n_map  # pose() = ... keeps the map
        ns, pose = register(K + 1)  # the drive goes on from the relocalised pose of frame K with frame K + 1's odometry
        assert ns > 0 and L.kfac_pipeline_num_map_points(p) >= n_map
        dt, ang = ko.pose_delta(pose, z["plain_poses"][K + 1])
        assert dt <= 0.05 and ang <= 0.01, (dt, ang)
        L.kfac_pipeline_set_pose(p, start.ctypes.data)
        assert L.kfac_pipeline_num_map_points(p) == 0  # the contrast: SetPose clears the map
    finally:
        L.kfac_pipeline_destroy(p)


def test_staged_frame_and_last_frame_survive_a_search(oracle, workload):
    """On one context with option "correspondences" 1: a frame registered, its clouds and correspondence report read, a search (host
    and device points) on the same map, the clouds and report read again (unchanged); then a frame staged, searched around, and
    registered: its pose, clouds, result block and the map (in key order) bit for bit those of a second context that never searched"""
    import torch

    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(2)
    ctxs = [kb.Context(0), kb.Context(0)]
    maps = []
    try:
        for c in ctxs:
            c.set_option("correspondences", 1)
            maps.append(_map(kb, c, w))
        ident = np.ascontiguousarray(ko.IDENTITY)
        scan = np.ascontiguousarray(w.scan[:8000], dtype=np.float64)
        src = _src(w, 1000)
        he, st = (0.2, 0.2, 0.02), (0.1, 0.1, 0.02)
        kw = dict(max_range=100.0, min_range=0.0, deskew=False, voxel_size=w.voxel_size)

        def snapshot(c):
            f, s = kb.frame_clouds_device(c)
            return (torch.as_tensor(f, device="cuda").cpu().numpy().copy(), torch.as_tensor(s, device="cuda").cpu().numpy().copy(),
                    kb.frame_correspondences(c))

        outs = []
        for j, (c, gm) in enumerate(zip(ctxs, maps)):
            first = kb.RegisterStagedFrame(gm, kb.StageFrame(c, scan), ident, ident, w.prior, ident, w.tau, **kw)
            if j == 0:
                before = snapshot(c)
                assert before[2].n_inliers > 0
                gm.PoseSearch(src, first[0], 0.3, he, st, levels=2, keep=4)
                gm.PoseSearch(torch.from_numpy(src).cuda(), first[0], 0.3, he, st, levels=2, keep=4)
                after = snapshot(c)
                assert all(np.array_equal(x, y) for x, y in zip(before[:2], after[:2])) and before[2] == after[2]
            staged = kb.StageFrame(c, scan)
            if j == 0:
                gm.PoseSearch(src, first[0], 0.3, he, st, levels=2, keep=4)
            outs.append(kb.RegisterStagedFrame(gm, staged, ident, ident, first[0], ident, w.tau, **kw))
        (a, b) = outs
        assert np.array_equal(a[0], b[0])
        assert np.array_equal(np.asarray(a[1]), np.asarray(b[1])) and np.array_equal(np.asarray(a[2]), np.asarray(b[2]))
        import ctypes as C
        assert C.string_at(C.addressof(a[3]), C.sizeof(a[3])) == C.string_at(C.addressof(b[3]), C.sizeof(b[3]))
        from test_gpu_laserscan import same_map
        assert same_map(*maps)  # voxel content in key order (the order voxels are created in is not part of the result)
    finally:
        for gm in maps:
            gm.close()
        for c in ctxs:
            c.close()
