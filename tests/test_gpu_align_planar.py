"""The planar alignment on the GPU (kicp_map_align_planar, kicp_map_align_planar_device through VoxelHashMap.AlignPlanar) against the
oracle's restatement (tests/align_planar_oracle.py): cfg2 bit for bit (pose, status, iterations, report) and the report against
Correspondences at the returned pose; recovery of a known planar perturbation of cfg2's true pose by PoseSearch and then AlignPlanar of
its kept hypotheses; host, device float64 and strided float32 device inputs; repeated and batched calls; no side effect on the map or
the last frame's report; the C++ facade against the C call."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import align_planar_oracle as AO

pytestmark = pytest.mark.gpu


def _map(kb, ctx, w):
    gm = kb.VoxelHashMap(ctx, w.voxel_size, w.max_range, w.max_points_per_voxel)
    gm.load_voxels(*w.map.export_voxels())
    return gm


def _src(w, n):
    return np.ascontiguousarray(w.scan[:: max(1, len(w.scan) // n)][:n], dtype=np.float64)


def _starts(ko, w):
    return np.array([w.prior, ko.se3_compose(w.true_pose, ko.planar_pose(0.13, -0.07, 0.015)),
                     ko.se3_compose(w.true_pose, ko.planar_pose(-0.05, 0.11, -0.02))])


def test_cfg2_against_oracle_and_correspondences(oracle, workload):
    """three starts on cfg2 at the registration's gate and a narrow one: every result the oracle's bit for bit; its count the
    Correspondences report's at the returned pose and its sum_sq within 1e-12 of that report's"""
    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(2)
    ctx = kb.Context(0)
    gm = _map(kb, ctx, w)
    try:
        src = _src(w, 3000)
        starts = _starts(ko, w)
        for tau in (w.tau, 0.3):
            got = gm.AlignPlanar(src, starts, tau)
            assert len(got) == 3
            for a, T0 in zip(got, starts):
                AO.check_alignment(a, AO.align(ko, w.map, src, T0, tau), tau)
                _, dist, inl, cs = gm.Correspondences(src, a.pose, tau)
                assert cs.n_inliers == a.n_inliers > 0 and int(inl.sum()) == a.n_inliers
                assert abs(cs.sum_sq - a.sum_sq) <= 1e-12 * abs(cs.sum_sq)
                assert a.iterations > 0 and a.status in (kb._capi.KICP_ALIGN_CONVERGED, kb._capi.KICP_ALIGN_MAX_ITERATIONS)
    finally:
        gm.close()
        ctx.close()


def _planar_error(ko, pose, truth):
    """|x|, |y|, |yaw| of truth^-1 * pose"""
    d = ko.se3_compose(ko.se3_inverse(truth), np.asarray(pose, dtype=np.float64))
    return np.abs(np.array([d[4], d[5], 2.0 * math.atan2(d[2], d[3])]))


def test_recovery_search_then_align(oracle, workload):
    """a prior perturbed from cfg2's true pose by a known off-lattice (x, y, yaw); PoseSearch (3 levels, finest steps 0.05 m and
    0.01 rad, keep 8, gate 0.15 m), then AlignPlanar of the 8 kept poses with the same gate, the best picked by (stopped normally,
    more inliers, smaller sum_sq).  Every result is the oracle's bit for bit, and the pick is within half a finest step of the truth on
    every axis: the oracle's run on the CPU gives (0.0025 m, 0.011 m, 0.00015 rad) against the search's best (0.010 m, 0.0054 m,
    0.001 rad)."""
    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(2)
    ctx = kb.Context(0)
    gm = _map(kb, ctx, w)
    try:
        src = _src(w, 2000)
        prior = ko.se3_compose(w.true_pose, ko.planar_pose(0.37, -0.23, 0.041))
        st, levels = (0.2, 0.2, 0.04), 3
        hyps, _ = gm.PoseSearch(src, prior, 0.15, (0.8, 0.8, 0.08), st, levels=levels, keep=8)
        starts = np.array([h.pose for h in hyps])
        got = gm.AlignPlanar(src, starts, 0.15)
        for a, T0 in zip(got, starts):
            AO.check_alignment(a, AO.align(ko, w.map, src, T0, 0.15))
        ok = (kb._capi.KICP_ALIGN_CONVERGED, kb._capi.KICP_ALIGN_MAX_ITERATIONS)
        best = min(got, key=lambda a: (a.status not in ok, -a.n_inliers, a.sum_sq))
        fine = np.array(st) / 2 ** (levels - 1)
        err = _planar_error(ko, best.pose, w.true_pose)
        assert (err < fine / 2).all(), (err, fine)
    finally:
        gm.close()
        ctx.close()


def test_inputs_repeat_batch_and_no_side_effects(oracle, workload):
    """host float64, device float64 and strided float32 device records give the same bits (float32 points widened exactly); a
    repeated call the same bits; each start alone the bits of the batched call; the map's export_voxels unchanged"""
    import torch

    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(2)
    ctx = kb.Context(0)
    gm = _map(kb, ctx, w)
    try:
        src = _src(w, 1500).astype(np.float32).astype(np.float64)
        starts = _starts(ko, w)
        before = gm.export_voxels()
        a = gm.AlignPlanar(src, starts, 0.3)
        b = gm.AlignPlanar(src, starts, 0.3)
        c = gm.AlignPlanar(torch.from_numpy(src).cuda(), starts, 0.3)
        rec = torch.zeros((len(src), 5), dtype=torch.float32, device="cuda")
        rec[:, 1:4] = torch.from_numpy(src.astype(np.float32)).cuda()
        e = gm.AlignPlanar(rec, starts, 0.3, point_step=20, offsets=(4, 8, 12))
        one = [gm.AlignPlanar(src, T0, 0.3)[0] for T0 in starts]
        for got in (b, c, e, one):
            assert len(got) == len(a)
            for x, y in zip(got, a):
                assert np.array_equal(x.pose, y.pose) and x[1:] == y[1:]
        AO.check_alignment(a[1], AO.align(ko, w.map, src, starts[1], 0.3))
        many = gm.AlignPlanar(src, np.tile(starts, (22, 1))[:64], 0.3)
        assert len(many) == 64 and all(np.array_equal(x.pose, a[k % 3].pose) and x[1:] == a[k % 3][1:] for k, x in enumerate(many))
        after = gm.export_voxels()
        assert all(np.array_equal(x, y) for x, y in zip(before, after))
    finally:
        gm.close()
        ctx.close()


def test_last_frame_report_survives_an_alignment(oracle, workload):
    """with option "correspondences" 1: a frame registered, its clouds and correspondence report read, an alignment (host and device
    points) on the same map, the clouds and report read again: unchanged"""
    import torch

    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(2)
    ctx = kb.Context(0)
    ctx.set_option("correspondences", 1)
    gm = _map(kb, ctx, w)
    try:
        ident = np.ascontiguousarray(ko.IDENTITY)
        scan = np.ascontiguousarray(w.scan[:8000], dtype=np.float64)
        kw = dict(max_range=100.0, min_range=0.0, deskew=False, voxel_size=w.voxel_size)
        first = kb.RegisterStagedFrame(gm, kb.StageFrame(ctx, scan), ident, ident, w.prior, ident, w.tau, **kw)

        def snapshot():
            f, s = kb.frame_clouds_device(ctx)
            return (torch.as_tensor(f, device="cuda").cpu().numpy().copy(), torch.as_tensor(s, device="cuda").cpu().numpy().copy(),
                    kb.frame_correspondences(ctx))

        before = snapshot()
        assert before[2].n_inliers > 0
        vox = gm.export_voxels()
        src = _src(w, 1000)
        gm.AlignPlanar(src, first[0], 0.3)
        gm.AlignPlanar(torch.from_numpy(src).cuda(), [first[0], w.prior], 0.3)
        after = snapshot()
        assert all(np.array_equal(x, y) for x, y in zip(before[:2], after[:2])) and before[2] == after[2]
        assert all(np.array_equal(x, y) for x, y in zip(vox, gm.export_voxels()))
    finally:
        gm.close()
        ctx.close()


def test_facade_align_planar_equals_c_call(oracle, workload):
    """kiss_icp::VoxelHashMap::AlignPlanar (tests/hooks/align_planar_hooks.cpp) == kicp_map_align_planar on the same map: every field
    bit for bit except the pose, which passes through Sophus (from_pose7 normalises the quaternion again) and agrees to 1e-15"""
    from kinematic_icp_b200 import _capi
    ko = oracle
    w = workload(2)
    H = C.CDLL(os.path.join(os.path.dirname(os.path.abspath(__file__)), "hooks", "_build", "libkicp_align_planar_hooks.so"))
    H.kfal_map_create.restype = C.c_void_p
    H.kfal_map_create.argtypes = [C.c_double, C.c_double, C.c_uint]
    H.kfal_map_destroy.argtypes = [C.c_void_p]
    H.kfal_map_add_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    H.kfal_map_handle.restype = C.c_void_p
    H.kfal_map_handle.argtypes = [C.c_void_p]
    H.kfal_map_align_planar.restype = C.c_int32
    H.kfal_map_align_planar.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.POINTER(AO.Params),
                                        C.POINTER(AO.Alignment)]
    lib = _capi.lib()
    m = H.kfal_map_create(w.voxel_size, w.max_range, w.max_points_per_voxel)
    try:
        pts = np.ascontiguousarray(w.map.pointcloud(), dtype=np.float64)
        H.kfal_map_add_points(m, pts.ctypes.data, len(pts))
        src = _src(w, 1500)
        starts = np.ascontiguousarray(_starts(ko, w))
        p = AO.Params(0.3, 1e-3, 10)
        a = (AO.Alignment * 3)()
        assert H.kfal_map_align_planar(m, src.ctypes.data, len(src), starts.ctypes.data, 3, C.byref(p), a) == 3
        b = (AO.Alignment * 3)()
        _capi.check(lib.kicp_map_align_planar(C.c_void_p(H.kfal_map_handle(m)), _capi.dp(src), len(src), _capi.dp(starts), 3,
                                              C.cast(C.byref(p), C.POINTER(_capi.PlanarAlignParams)),
                                              C.cast(b, C.POINTER(_capi.PlanarAlignment))), "kicp_map_align_planar")
        for x, y in zip(a, b):
            assert np.abs(np.array(x.pose[:]) - np.array(y.pose[:])).max() <= 1e-15
            assert bytes(x)[C.sizeof(C.c_double) * 7:] == bytes(y)[C.sizeof(C.c_double) * 7:]
        assert b[0].n_inliers > 0
    finally:
        H.kfal_map_destroy(m)
