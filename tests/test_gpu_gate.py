"""The gate scenes and the non-finite registrations of tests/gate_scenes.py on the H100 (the emulator's counterpart is
tests/test_gate_emu_cpu.py).  kicp_register.cu is compiled with FMA contraction, so only here does the device's own arithmetic decide
the gate: N of the first pass must be the oracle's and the scene's own count at every point whose reference norm is prev(tau), tau
or next(tau) — through kicp_register (host pointer: chunked upload overlapped with the kernel), kicp_register_points (float32),
kicp_register_scan_async and kicp_register_frame, on every launch shape."""
import numpy as np
import pytest

import gate_scenes as G
from test_gpu_scenes import gpu_map

pytestmark = pytest.mark.gpu
TOL_T, TOL_R = 1e-6, 1e-7
# (persistent, nn_cache, ctas_per_sm)
SHAPES = [(p, c, k) for p in (1, 0) for c in (0, 1, 2) for k in (0, 1)]


@pytest.fixture(scope="module")
def gate_scenes(oracle):
    return G.gate_scenes(oracle)


@pytest.fixture(scope="module")
def nonfinite_scenes(oracle):
    return G.nonfinite_reg_scenes(oracle)


def shapes(ctx, run):
    try:
        for persistent, cache, ctas in SHAPES:
            ctx.set_option("persistent", persistent)
            ctx.set_option("nn_cache", cache)
            ctx.set_option("ctas_per_sm", ctas)
            run((persistent, cache, ctas))
    finally:
        ctx.set_option("persistent", 1)
        ctx.set_option("nn_cache", 1)
        ctx.set_option("ctas_per_sm", 0)


def entry_points(kb, ctx, gm, scan, last, odom, tau, kw):
    """(name, RegResult) of one registration of `scan` through each entry point that takes it as it is."""
    reg = kb.KinematicRegistration(kw.get("max_iter", 10), kw.get("conv", 1e-3), 1, kw.get("adaptive", True), kw.get("fixed_reg", 0.0))
    out = []
    reg.ComputeRobotMotion(scan, gm, last, odom, tau)
    out.append(("kicp_register_points" if scan.dtype == np.float32 else "kicp_register", reg.last_result))
    if scan.dtype == np.float64:
        ds = kb.Scan(ctx, len(scan))
        try:
            ds.upload(scan)
            r = kb.pinned_result()
            reg.enqueue(ds, gm, last, odom, tau, r)
            ctx.synchronize()
            out.append(("kicp_register_scan_async", r))
        finally:
            ds.close()
    return out


def test_gate_first_pass_matches_reference_gpu(oracle, gpu_ctx, gate_scenes):
    """N of the first pass exactly (the oracle's, and the scene's own count), the sums to 1e-9, the pose."""
    import kinematic_icp_b200 as kb
    ko = oracle
    for sc in gate_scenes:
        po, st = sc.om.register(np.asarray(sc.scan, dtype=np.float64), sc.last, sc.odom, sc.tau, **sc.kw)
        assert st.sums_np()[0, 5] == sc.expected_n, sc.name
        gm = gpu_map(kb, gpu_ctx, sc.voxel_size, sc.cap, sc.voxels)

        def run(shape):
            for name, res in entry_points(kb, gpu_ctx, gm, sc.scan, sc.last, sc.odom, sc.tau, sc.kw):
                where = (sc.name, name, shape)
                assert res.sums_np()[0, 5] == sc.expected_n, where + (res.sums_np()[0, 5],)
                assert res.iterations == st.iterations, where
                assert np.allclose(res.sums_np()[:, :5], st.sums_np()[:, :5], rtol=1e-9, atol=1e-9), where
                dt, ang = ko.pose_delta(res.pose_np(), po)
                assert dt <= TOL_T and ang <= TOL_R, where + (dt, ang)
        try:
            shapes(gpu_ctx, run)
        finally:
            gm.close()


def test_gate_through_the_frame_path_gpu(oracle, gpu_ctx, gate_scenes):
    """kicp_register_frame with one iteration, identity lidar_to_base, no de-skew and min_range 0: the scan's points are 4 voxels
    of the map apart, so both down-samples return the scan itself, and N of the first pass is the scene's."""
    import kinematic_icp_b200 as kb
    ko = oracle
    for sc in gate_scenes:
        scan = np.asarray(sc.scan, dtype=np.float64)
        gm = gpu_map(kb, gpu_ctx, sc.voxel_size, sc.cap, sc.voxels)
        try:
            pose, frame, source, res = kb.RegisterFrame(
                gm, sc.scan, np.zeros(0), ko.IDENTITY, ko.IDENTITY, sc.last, sc.odom, sc.tau, max_range=1e9, min_range=0.0, deskew=False,
                voxel_size=sc.voxel_size, max_num_iterations=1, use_adaptive_odometry_regularization=sc.kw.get("adaptive", True),
                fixed_regularization=sc.kw.get("fixed_reg", 0.0))
        finally:
            gm.close()
        assert np.array_equal(frame, scan) and np.array_equal(source, scan), sc.name
        assert res.sums_np()[0, 5] == sc.expected_n, (sc.name, res.sums_np()[0, 5])


def test_nonfinite_points_match_reference_gpu(oracle, gpu_ctx, nonfinite_scenes):
    """NaN, +-Inf and +-3e9 vs scan points (float64 and float32), a map with non-finite points and NaN-first voxels: N of every pass,
    no NaN in the sums, the pose.  tau = 1e12: N of the first pass and its sums (to 1e-9 of the largest)."""
    import kinematic_icp_b200 as kb
    ko = oracle
    for sc in nonfinite_scenes:
        huge = sc.kw.get("huge", False)
        kw = {k: v for k, v in sc.kw.items() if k != "huge"}
        gm = gpu_map(kb, gpu_ctx, sc.voxel_size, sc.cap, sc.voxels)
        try:
            for scan in (sc.scan, sc.scan.astype(np.float32)):
                po, st = sc.om.register(np.asarray(scan, dtype=np.float64), sc.last, sc.odom, sc.tau, **kw)
                want = st.sums_np()[:, :6]

                def run(shape):
                    for name, res in entry_points(kb, gpu_ctx, gm, scan, sc.last, sc.odom, sc.tau, kw):
                        where = (sc.name, name, str(scan.dtype), shape)
                        got = res.sums_np()[:, :6]
                        assert not np.isnan(got[:len(want)]).any(), where
                        if huge:
                            assert got[0, 5] == want[0, 5] > 0, where
                            assert np.all(np.abs(got[0, :5] - want[0, :5]) <= 1e-9 * np.abs(want[0, :5]).max()), where
                            continue
                        assert res.iterations == st.iterations, where
                        assert np.array_equal(got[:, 5], want[:, 5]), where
                        scale = np.abs(want[:, :5]).max(axis=1, keepdims=True)
                        assert np.all(np.abs(got[:, :5] - want[:, :5]) <= 1e-9 * scale), where
                        dt, ang = ko.pose_delta(res.pose_np(), po)
                        assert dt <= TOL_T and ang <= TOL_R, where + (dt, ang)
                shapes(gpu_ctx, run)
        finally:
            gm.close()
