"""The edge scenes of tests/scenes.py on the H100 (the emulator's counterpart is tests/test_edges_emu_cpu.py): points on voxel faces,
norms equal to the range gate, candidates exactly map_resolution from a stored point, first points exactly max_distance away,
probe chains of colliding keys that wrap past the last slot, the de-skew edges, and NaN / +-Inf / +-huge coordinates.  The device
converts a floored coordinate with its own instruction (cvt.rzi.s32.f64 gives 0 for NaN and INT_MAX above the int range), so only
these tests see whether its voxel keys are the reference's (INT_MIN for all of those, as on x86-64).  Floats are compared by bit
pattern, so NaN equals NaN."""
import numpy as np
import pytest

import scenes as S
from test_edges_emu_cpu import deskew_cases, sorted_voxels
from test_gpu_scenes import check, every_launch, gpu_map

pytestmark = pytest.mark.gpu
DBL_MAX = np.finfo(np.float64).max


def assert_same_map(gm, om):
    assert gm.num_points() == om.num_points() and gm.num_voxels() == om.num_voxels()
    k1, c1, p1 = sorted_voxels(*gm.export_voxels())
    k0, c0, p0 = sorted_voxels(*om.export_voxels())
    assert np.array_equal(k1, k0) and np.array_equal(c1, c0) and S.same_bits(p1, p0)


def test_downsample_boundary_clouds_gpu(oracle, gpu_ctx):
    import kinematic_icp_b200 as kb
    ko = oracle
    for vs, pts, _, _ in S.boundary_clouds():
        assert S.same_bits(kb.VoxelDownsample(gpu_ctx, pts, vs), ko.voxel_downsample(pts, vs)), vs


def test_downsample_nonfinite_gpu(oracle, gpu_ctx):
    """NaN / Inf / huge points: a NaN point first in voxel (0, 0, 0) must not replace that voxel's survivor, +huge and +Inf points
    share the INT_MIN voxel with -huge ones."""
    import kinematic_icp_b200 as kb
    ko = oracle
    for vs in (0.5, 0.37, 1.5):
        cloud = S.with_nonfinite(np.random.default_rng(3).uniform(-2, 2, (500, 3)) * vs, vs)
        ref = ko.voxel_downsample(cloud, vs)
        assert S.same_bits(kb.VoxelDownsample(gpu_ctx, cloud, vs), ref), vs


@pytest.mark.parametrize("min_range,max_range", [(3.25, 104.0), (0.0, 13.0)])
def test_preprocess_range_gate_gpu(oracle, gpu_ctx, min_range, max_range):
    import kinematic_icp_b200 as kb
    ko = oracle
    pts, norms = S.range_gate_cloud(min_range if min_range else 13.0 / 16, max_range)
    assert (norms == max_range).sum() >= 7
    pts = np.concatenate([pts, S.nonfinite_rows(1.0)])
    ref = ko.preprocess(pts, np.zeros(0), ko.IDENTITY, max_range, min_range, False)
    assert 0 < len(ref) < len(pts)
    assert S.same_bits(kb.Preprocess(gpu_ctx, pts, np.zeros(0), ko.IDENTITY, max_range, min_range, False), ref)


def test_preprocess_deskew_edges_gpu(oracle, gpu_ctx, workload):
    """Here the log of the motion is the library's own (se3_log_host): its small-angle branch, and its qw < 0 branch near pi."""
    import kinematic_icp_b200 as kb
    ko = oracle
    scan = np.concatenate([workload(2).scan] * 3)
    for name, motion, stamps_of in deskew_cases(ko):
        for pts in (scan, scan[:1]):
            stamps = stamps_of(len(pts))
            out = kb.Preprocess(gpu_ctx, pts, stamps, motion, 100.0, 0.5, True)
            ref = ko.preprocess(pts, stamps, motion, 100.0, 0.5, True)
            assert out.shape == ref.shape, name
            if len(ref):
                assert np.abs(out - ref).max() < 1e-12, name


@pytest.mark.parametrize("cap", [4, 16])
def test_addpoints_exact_map_resolution_gpu(oracle, gpu_ctx, cap):
    import kinematic_icp_b200 as kb
    ko = oracle
    pts, exact, closer = S.map_rule_points(cap=cap)
    assert exact > 0 and closer > 0
    for seq in (pts, S.with_nonfinite(pts, 1.0)):
        om, gm = ko.OracleMap(1.0, 100.0, cap), kb.VoxelHashMap(gpu_ctx, 1.0, 100.0, cap)
        try:
            om.add_points(seq)
            gm.AddPoints(seq)
            assert_same_map(gm, om)
        finally:
            gm.close()


@pytest.mark.parametrize("cap", [1, 255])
def test_addpoints_fills_extreme_caps_gpu(oracle, gpu_ctx, cap):
    import kinematic_icp_b200 as kb
    ko = oracle
    rng = np.random.default_rng(cap)
    g = (np.stack(np.meshgrid(*[np.arange(7)] * 3, indexing="ij"), -1).reshape(-1, 3) + 0.5) / 7.0
    pts = np.concatenate([(g[rng.permutation(len(g))] + [2, -3, 1]) * 0.37, rng.uniform(0, 4, (600, 3)) * 0.37])
    om, gm = ko.OracleMap(0.37, 100.0, cap), kb.VoxelHashMap(gpu_ctx, 0.37, 100.0, cap)
    try:
        for chunk in np.array_split(pts, 3):
            om.add_points(chunk)
            gm.AddPoints(chunk)
        assert_same_map(gm, om)
        assert om.export_voxels()[1].max() == cap
    finally:
        gm.close()


def test_update_evicts_at_exactly_max_distance_gpu(oracle, gpu_ctx):
    import kinematic_icp_b200 as kb
    ko = oracle
    pts, sq = S.far_first_points()
    assert (sq == 144.0).any() and (sq < 144.0).any()
    for seq in (pts, S.with_nonfinite(pts, 3.0)):
        om, gm = ko.OracleMap(3.0, 12.0, 8), kb.VoxelHashMap(gpu_ctx, 3.0, 12.0, 8)
        try:
            om.update_origin(seq, np.zeros(3))
            gm.Update(seq, np.zeros(3))
            assert_same_map(gm, om)
            om.update_pose(seq, ko.planar_pose(0.0, 0.0, 0.0))
            gm.Update(seq, ko.planar_pose(0.0, 0.0, 0.0))
            assert_same_map(gm, om)
        finally:
            gm.close()


def test_addpoints_nonfinite_gpu(oracle, gpu_ctx):
    """A NaN point takes a slot of the INT_MIN voxel, not of voxel (0, 0, 0), where a real point the reference keeps would then find
    the voxel full; a NaN first point of voxel (0, 0, 0) would never be evicted."""
    import kinematic_icp_b200 as kb
    ko = oracle
    rng = np.random.default_rng(4)
    for vs, cap in ((0.5, 2), (0.37, 1), (1.0, 20)):
        seq = S.with_nonfinite(rng.uniform(-3, 3, (800, 3)), vs)
        om, gm = ko.OracleMap(vs, 4.0, cap), kb.VoxelHashMap(gpu_ctx, vs, 4.0, cap)
        try:
            om.add_points(seq)
            gm.AddPoints(seq)
            assert_same_map(gm, om)
            om.update_origin(seq[:50], np.array([3.0, 0.0, 0.0]))
            gm.Update(seq[:50], np.array([3.0, 0.0, 0.0]))
            assert_same_map(gm, om)
        finally:
            gm.close()


def test_nearest_nonfinite_queries_gpu(oracle, gpu_ctx):
    """+huge queries must find the points of the INT_MIN voxel, as the reference does; NaN / Inf queries find nothing."""
    import kinematic_icp_b200 as kb
    ko = oracle
    vs = 0.5
    rng = np.random.default_rng(5)
    pts = np.concatenate([rng.uniform(-2, 2, (400, 3)), [[-3e9 * vs, 0.1, 0.1], [-3e9 * vs, -3e9 * vs, -3e9 * vs]]])
    om, gm = ko.OracleMap(vs, 100.0, 20), kb.VoxelHashMap(gpu_ctx, vs, 100.0, 20)
    try:
        om.add_points(pts)
        gm.AddPoints(pts)
        q = S.with_nonfinite(rng.uniform(-2, 2, (200, 3)), vs)
        pg, dg = gm.GetClosestNeighbor(q)
        po, do = om.nearest(q)
        assert S.same_bits(dg, do) and S.same_bits(pg, po)
        assert (do[np.all(q == 3e9 * vs, axis=1)] < DBL_MAX).all()
    finally:
        gm.close()


def test_colliding_keys_gpu(oracle, gpu_ctx):
    """Chains of 3 to 40 colliding voxels that wrap past slot 0: find-or-create under same-warp collisions, k_add_commit's search
    for its own slot, k_nearest and the registration kernel's long-chain loop, through every launch shape."""
    import kinematic_icp_b200 as kb
    ko = oracle
    for sc in S.collision_scenes(ko):
        pts = sc.om.export_voxels()[2]
        om, gm = ko.OracleMap(sc.voxel_size, S.FAR, sc.cap + 3), kb.VoxelHashMap(gpu_ctx, sc.voxel_size, 20.0 * sc.voxel_size, sc.cap + 3)
        try:
            om.add_points(pts[::2])
            gm.AddPoints(pts[::2])
            extra = np.concatenate([pts[1::2], S.with_nonfinite(sc.scan[:50], sc.voxel_size)])
            om.add_points(extra)
            gm.AddPoints(extra)
            assert_same_map(gm, om)
            q = S.with_nonfinite(sc.scan, sc.voxel_size)
            pg, dg = gm.GetClosestNeighbor(q)
            po, do = om.nearest(q)
            assert S.same_bits(dg, do) and S.same_bits(pg, po), sc.name
        finally:
            gm.close()
        gm = gpu_map(kb, gpu_ctx, sc.voxel_size, sc.cap, sc.voxels)
        try:
            every_launch(gpu_ctx, lambda: check(ko, kb, sc.om, gm, sc.scan, sc.last, sc.odom, sc.tau, **sc.kw))
            scan = S.with_nonfinite(sc.scan, sc.voxel_size)
            every_launch(gpu_ctx, lambda: check(ko, kb, sc.om, gm, scan, sc.last, sc.odom, sc.tau, max_iter=1))
        finally:
            gm.close()
