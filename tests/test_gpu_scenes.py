"""The scenes of tests/scenes.py on the H100: ties and ulp-level near-ties of the nearest-neighbour choice, map shapes the
workloads never use, and the 40 randomised scenes whose reference poses are tests/golden/ref_fuzz.npz — through every launch
shape of the registration kernel and through the map kernels' GetClosestNeighbor."""
import os

import numpy as np
import pytest

import scenes as S

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL_T, TOL_R = 1e-6, 1e-7
# (persistent, nn_cache): 0 = no certificates, 1 = by scan size, 2 = always (these scans are small: 2 is what turns them on)
LAUNCHES = [(1, 0), (1, 1), (1, 2), (0, 0)]


def gpu_map(kb, ctx, voxel_size, cap, voxels):
    gm = kb.VoxelHashMap(ctx, voxel_size, S.FAR, cap)
    gm.load_voxels(*voxels)
    return gm


def check(ko, kb, om, gm, scan, last, odom, tau, max_iter=10, conv=1e-3, adaptive=True, fixed_reg=0.0):
    reg = kb.KinematicRegistration(max_iter, conv, 1, adaptive, fixed_reg)
    pose = reg.ComputeRobotMotion(scan, gm, last, odom, tau)
    po, st = om.register(scan, last, odom, tau, max_iter=max_iter, conv=conv, adaptive=adaptive, fixed_reg=fixed_reg)
    res = reg.last_result
    assert np.array_equal(np.isnan(pose), np.isnan(po))
    if np.isnan(po).any():  # no correspondence: the reference iterates on with a NaN pose, the device stops and says so
        assert res.status == kb.KICP_WARN_NO_CORRESPONDENCES and res.sums_np()[0, 5] == st.sums_np()[0, 5] == 0
        return pose
    dt, ang = ko.pose_delta(pose, po)
    assert dt <= TOL_T and ang <= TOL_R, (dt, ang)
    assert res.iterations == st.iterations
    assert np.array_equal(res.sums_np()[:, 5], st.sums_np()[:, 5])
    assert np.allclose(res.sums_np()[:, :5], st.sums_np()[:, :5], rtol=1e-9, atol=1e-9)
    return pose


def every_launch(ctx, run):
    try:
        for persistent, cache in LAUNCHES:
            ctx.set_option("persistent", persistent)
            ctx.set_option("nn_cache", cache)
            run()
    finally:
        ctx.set_option("persistent", 1)
        ctx.set_option("nn_cache", 1)


def test_neighbour_ties_match_reference_gpu(oracle, gpu_ctx):
    import kinematic_icp_b200 as kb
    ko = oracle
    for sc in S.tie_scenes(ko):
        gm = gpu_map(kb, gpu_ctx, sc.voxel_size, sc.cap, sc.voxels)
        try:
            q = sc.queries(ko)
            pg, dg = gm.GetClosestNeighbor(q)
            po, do = sc.om.nearest(q)
            assert np.array_equal(dg, do) and np.array_equal(pg, po), sc.name
            every_launch(gpu_ctx, lambda: check(ko, kb, sc.om, gm, sc.scan, sc.last, sc.odom, sc.tau, **sc.kw))
        finally:
            gm.close()


def test_map_shapes_match_oracle_gpu(oracle, gpu_ctx):
    import kinematic_icp_b200 as kb
    ko = oracle
    for sc in S.shape_scenes(ko):
        assert np.frexp(sc.voxel_size)[0] != 0.5 and np.all(sc.voxels[1] == sc.cap)
        gm = gpu_map(kb, gpu_ctx, sc.voxel_size, sc.cap, sc.voxels)
        try:
            every_launch(gpu_ctx, lambda: check(ko, kb, sc.om, gm, sc.scan, sc.last, sc.odom, sc.tau, **sc.kw))
        finally:
            gm.close()


def test_fuzz_scenes_vs_reference_gpu(oracle, gpu_ctx):
    """All 40 scenes, each through one launch shape in turn, against the oracle (N per pass, sums) and the reference's poses."""
    import kinematic_icp_b200 as kb
    ko = oracle
    ref = np.load(os.path.join(GOLDEN, "ref_fuzz.npz"))["poses"]
    try:
        for case, (om, vs, cap, _, scan, last, odom, tau, kw) in enumerate(S.fuzz_cases(ko)):
            persistent, cache = LAUNCHES[case % len(LAUNCHES)]
            gpu_ctx.set_option("persistent", persistent)
            gpu_ctx.set_option("nn_cache", cache)
            gm = gpu_map(kb, gpu_ctx, vs, cap, om.export_voxels())
            try:
                pose = check(ko, kb, om, gm, scan, last, odom, tau, **kw)
            finally:
                gm.close()
            assert np.array_equal(np.isnan(pose), np.isnan(ref[case])), (case, kw)
            if not np.isnan(pose).any():
                dt, ang = ko.pose_delta(pose, ref[case])
                assert dt <= TOL_T and ang <= TOL_R, (case, kw, dt, ang)
    finally:
        gpu_ctx.set_option("persistent", 1)
        gpu_ctx.set_option("nn_cache", 1)
    assert case == 39
