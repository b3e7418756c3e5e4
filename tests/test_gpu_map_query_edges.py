"""The edge scenes of the three map queries (correspondences, pose search, planar alignment) on the H100, against the oracles the SIMT
emulator's tests use (tests/test_{correspondences,pose_search,align_planar}_emu_cpu.py).  Only here are the kernels nvcc's -fmad=false
code, with the device's own sqrt and division inside voxel_coord and the pruning margin of lane_gated_neighbor: the gate scenes (the far
origin and the exact (3, 4, 12) 2^k cases included), cfg2 moved by a dyadic offset near (2^19, 2^22, 0), the tie scenes, an empty map,
n = 0, non-finite points, a NaN pose, yaws at +-pi, a start without inliers, one iteration, a collinear cloud and voxels full to caps
1, 24, 25, 29 and 255.  Every scene goes through the host entry point, the device entry point and, where its points are
float32-representable, strided float32 records; the device maps are loaded from the oracle map's voxels."""
import math

import numpy as np
import pytest

import align_planar_oracle as AO
import gate_scenes as G
import pose_search_oracle as PO
import scenes as S
from corr_oracle import check_stats, oracle_corr
from test_gpu_correspondences import st_c
from test_gpu_scenes import gpu_map

pytestmark = pytest.mark.gpu
DBL_MAX = np.finfo(np.float64).max


def _map(kb, ctx, om):
    keys, counts, pts = om.export_voxels()
    if len(counts):
        return gpu_map(kb, ctx, om.voxel_size, om.max_points_per_voxel, (keys, counts, pts))
    return kb.VoxelHashMap(ctx, om.voxel_size, S.FAR, om.max_points_per_voxel)


def _inputs(src):
    """(name, points, keyword arguments): host float64, device float64 and, when every coordinate is a float32, strided float32
    records (x, y, z at bytes 4, 8, 12 of 20)"""
    import torch
    out = [("host", src, {}), ("device", torch.from_numpy(src).cuda(), {})]
    f32 = src.astype(np.float32)
    if np.array_equal(f32.astype(np.float64), src, equal_nan=True):
        rec = np.zeros((len(src), 5), np.float32)
        rec[:, 1:4] = f32
        out.append(("f32-records", torch.from_numpy(rec.view(np.uint8).reshape(-1)).cuda(), dict(point_step=20, offsets=(4, 8, 12))))
    return out


def _np(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)


def corr(ko, gm, om, src, pose, tau, name):
    """per-point neighbours, distances and inlier mask bit for bit, the counts exactly and the sums to 1e-12"""
    src = np.ascontiguousarray(src, dtype=np.float64).reshape(-1, 3)
    po, do, io, want = oracle_corr(ko, om, src, pose, tau)
    for kind, pts, kw in _inputs(src):
        p, d, inl, st = gm.Correspondences(pts, pose, tau, **kw)
        p, d, inl = _np(p), _np(d), _np(inl)
        where = (name, kind)
        assert S.same_bits(d, do) and S.same_bits(p, po), where
        assert np.array_equal(inl.astype(bool), io) and set(np.unique(inl)) <= {0, 1}, where
        check_stats(st_c(st), want)
    return want


def search(ko, gm, om, src, prior, tau, half_extent, step, levels, keep, name):
    """lattice points, levels and counts exactly, sum_sq bit for bit in the kernel's order, pose bits"""
    src = np.ascontiguousarray(src, dtype=np.float64).reshape(-1, 3)
    res = PO.search(ko, om, src, prior, tau, half_extent, step, levels, keep)
    for kind, pts, kw in _inputs(src):
        hyps, n_scored = gm.PoseSearch(pts, prior, tau, half_extent, step, levels=levels, keep=keep, **kw)
        assert n_scored == res["n_scored"], (name, kind)
        PO.check_hypotheses(hyps, res, np.asarray(prior, dtype=np.float64), len(src))
    return res


def align(ko, gm, om, src, starts, tau, max_iterations=10, convergence=1e-3, name=""):
    """every start's pose, status, iterations and report bit for bit"""
    src = np.ascontiguousarray(src, dtype=np.float64).reshape(-1, 3)
    starts = np.asarray(starts, dtype=np.float64).reshape(-1, 7)
    want = [AO.align(ko, om, src, T0, tau, max_iterations, convergence) for T0 in starts]
    for kind, pts, kw in _inputs(src):
        got = gm.AlignPlanar(pts, starts, tau, max_iterations, convergence, **kw)
        for a, (o, res) in enumerate(zip(got, want)):
            AO.check_alignment(o, res, (name, kind, a))
    return want


def pruned_share(ko, src, poses, tau, vs):
    """the share of the queries (src at each pose) for which lane_gated_neighbor probes fewer than 27 shifts: per axis the own key,
    +1 when key(q + tau + s) > key(q) and -1 when key(q - tau - s) < key(q), s = (|q| + tau) 2^-40 (ps_axis_shifts)"""
    q = np.concatenate([ko.se3_transform(np.asarray(p, dtype=np.float64), src) for p in poses])
    q = q[np.isfinite(q).all(1)]
    s = (np.abs(q) + tau) * 2.0 ** -40
    k, lo, hi = np.floor(q / vs), np.floor(((q - tau) - s) / vs), np.floor(((q + tau) + s) / vs)
    shifts = np.prod(1 + (hi >= k + 1) + (lo <= k - 1), axis=1)
    return float(np.mean(shifts < 27))


def test_gate_scenes(oracle, gpu_ctx):
    """every scene of G.gate_scenes (prev(tau), tau and next(tau) on voxel faces, edges and corners; the far origin (4.2e5, 5.8e6, 0);
    the exact (3, 4, 12) 2^k cases) with the emulator tests' source slices: the report of the whole scan (the inlier count the scene's
    own), the prior's hypothesis and its neighbours on a fine lattice, an alignment from the prior"""
    import kinematic_icp_b200 as kb
    ko = oracle
    for sc in G.gate_scenes(ko):
        gm = _map(kb, gpu_ctx, sc.om)
        try:
            src = np.asarray(sc.scan, dtype=np.float64)
            prior = ko.se3_compose(sc.last, sc.odom)
            want = corr(ko, gm, sc.om, src, prior, sc.tau, sc.name)
            assert want["n_inliers"] == sc.expected_n, sc.name
            search(ko, gm, sc.om, src[:150], prior, sc.tau, (1e-9, 1e-9, 1e-9), (1e-9, 1e-9, 1e-9), 2, 3, sc.name)
            align(ko, gm, sc.om, src[:150], [prior], sc.tau, max_iterations=3, name=sc.name)
            if "-far" in sc.name:
                assert pruned_share(ko, src[:150], [prior], sc.tau, sc.voxel_size) > 0.5
        finally:
            gm.close()


def test_far_from_the_origin(oracle, gpu_ctx, workload):
    """cfg2's map and scan on a 2^-20 grid, moved by (2^19 + 3/4, 2^22 - 5/8, 0) (exact), with its prior moved alike: all three
    queries at the registration's gate and at 0.3 m, and lane_gated_neighbor probing fewer than 27 shifts for most queries at 0.3 m"""
    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(2)
    off = np.array([2.0 ** 19 + 0.75, 2.0 ** 22 - 0.625, 0.0])
    grid = 2.0 ** 20
    mp = np.round(w.map.pointcloud() * grid) / grid
    assert np.array_equal((mp + off) - off, mp)
    om = ko.OracleMap(w.voxel_size, S.FAR, w.max_points_per_voxel)
    om.add_points(mp + off)
    gm = _map(kb, gpu_ctx, om)
    try:
        src = np.round(w.scan[::max(1, len(w.scan) // 1500)][:1500] * grid) / grid
        prior = np.array(w.prior, dtype=np.float64)
        prior[4:] += off
        moved = ko.se3_compose(prior, ko.planar_pose(0.13, -0.07, 0.015))
        for tau in (w.tau, 0.3):
            want = corr(ko, gm, om, src, prior, tau, "far-cfg2")
            assert 0 < want["n_inliers"] < len(src)
            res = align(ko, gm, om, src[:600], [prior, moved], tau, name="far-cfg2")
            assert all(r["v"][0] > 0 for r in res)
        res = search(ko, gm, om, src[:400], moved, 0.3, (0.2, 0.2, 0.04), (0.1, 0.1, 0.02), 3, 5, "far-cfg2")
        assert res["kept"][0][1] > 0
        share = pruned_share(ko, src[:400], [PO.pose(moved, res["u"], L)[0] for L, *_ in res["kept"]], 0.3, w.voxel_size)
        assert share > 0.5, share
    finally:
        gm.close()


def test_ties(oracle, gpu_ctx):
    """S.tie_scenes (exact and ulp-level near ties between voxels and inside one voxel) for all three queries with the emulator
    tests' slices and lattices, and the lattice of one repeated pattern whose score ties the rest of the key decides"""
    import kinematic_icp_b200 as kb
    ko = oracle
    for sc in S.tie_scenes(ko):
        gm = _map(kb, gpu_ctx, sc.om)
        try:
            src = np.asarray(sc.scan, dtype=np.float64)
            prior = ko.se3_compose(sc.last, sc.odom)
            corr(ko, gm, sc.om, src[:500], prior, sc.tau, sc.name)
            search(ko, gm, sc.om, src[:120], prior, sc.tau, (0.25, 0.25, 0.0), (0.125, 0.125, 0.1), 2, 6, sc.name)
            align(ko, gm, sc.om, src[:120], [prior], sc.tau, max_iterations=3, name=sc.name)
        finally:
            gm.close()
    grid = np.stack(np.meshgrid(np.arange(-4, 5), np.arange(-4, 5), [0.0], indexing="ij"), -1).reshape(-1, 3) + 0.5
    om = ko.OracleMap(1.0, S.FAR, 20)
    om.add_points(grid)
    gm = _map(kb, gpu_ctx, om)
    try:
        res = search(ko, gm, om, grid[20:40], ko.IDENTITY, 0.3, (2.0, 2.0, 0.0), (1.0, 1.0, 0.1), 1, 8, "lattice-ties")
        assert len({(c, s) for _, c, s, _ in res["kept"]}) < len(res["kept"])
    finally:
        gm.close()


def test_empty_map_n0_nonfinite_nan_pose_and_yaw_pi(oracle, gpu_ctx):
    """An empty map and n = 0 for all three (the alignment NO_CORRESPONDENCES after 0 iterations at the start's bits); non-finite
    source points for all three; a NaN pose for the report (every distance DBL_MAX, no inliers); levels and starts at yaw +-pi"""
    import kinematic_icp_b200 as kb
    ko = oracle
    vs = 0.5
    rng = np.random.default_rng(8)
    src = S.with_nonfinite(rng.uniform(-3, 3, (300, 3)), vs)
    pts = rng.uniform(-3, 3, (800, 3))
    start = ko.planar_pose(0.1, 0.05, 0.02)
    om = ko.OracleMap(vs, S.FAR, 20)
    gm = _map(kb, gpu_ctx, om)
    try:
        assert corr(ko, gm, om, src, ko.IDENTITY, 1.0, "empty")["n_inliers"] == 0
        res = search(ko, gm, om, src[:200], ko.IDENTITY, 1.0, (0.2, 0.2, 0.2), (0.1, 0.1, 0.1), 2, 7, "empty")
        assert [L for L, *_ in res["kept"]][:3] == [(0, 0, 0), (-1, 0, 0), (0, -1, 0)]
        res = align(ko, gm, om, pts[:100], [start], 0.4, name="empty")
        assert res[0]["status"] == AO.NO_CORRESPONDENCES and res[0]["iterations"] == 0 and res[0]["pose"] == list(start)
    finally:
        gm.close()
    om = ko.OracleMap(vs, S.FAR, 20)
    om.add_points(pts)
    gm = _map(kb, gpu_ctx, om)
    try:
        want = corr(ko, gm, om, src, ko.planar_pose(0.1, 0.05, 0.02), 0.4, "nonfinite")
        assert 0 < want["n_inliers"] < len(src)
        res = search(ko, gm, om, src[:200], ko.planar_pose(0.1, 0.05, 0.02), 0.4, (0.1, 0.1, 0.05), (0.05, 0.05, 0.05), 2, 4, "nonfinite")
        assert res["kept"][0][1] > 0
        res = align(ko, gm, om, S.with_nonfinite(pts[:200] + rng.normal(0, 0.02, (200, 3)), vs), [start, ko.IDENTITY], 0.4,
                    name="nonfinite")
        assert all(r["v"][0] > 0 for r in res)
        nan_pose = np.full(7, np.nan)
        want = corr(ko, gm, om, src, nan_pose, 0.4, "nan-pose")
        _, d, inl, st = gm.Correspondences(src, nan_pose, 0.4)
        assert want["n_inliers"] == 0 and (d == DBL_MAX).all() and not inl.any() and st.n_inliers == 0 and st.fitness == 0.0
        n0 = np.zeros((0, 3))
        corr(ko, gm, om, n0, ko.IDENTITY, 0.4, "n0")
        search(ko, gm, om, n0, ko.IDENTITY, 0.4, (0.1, 0.1, 0.1), (0.1, 0.1, 0.1), 2, 4, "n0")
        res = align(ko, gm, om, n0, [start], 0.4, name="n0")
        assert res[0]["status"] == AO.NO_CORRESPONDENCES and res[0]["iterations"] == 0 and res[0]["pose"] == list(start)
        search(ko, gm, om, pts[:60], ko.planar_pose(0.0, 0.0, 3.0), 0.4, (0.0, 0.0, np.pi), (0.1, 0.1, np.pi / 4), 2, 5, "yaw-pi")
        res = align(ko, gm, om, pts[:120], [ko.planar_pose(0.02, 0.0, math.pi), ko.planar_pose(0.0, 0.01, -math.pi),
                                            ko.planar_pose(0.0, 0.0, math.pi - 1e-3)], 0.4, max_iterations=4, name="yaw-pi")
        assert all(r["v"][0] > 0 for r in res)
    finally:
        gm.close()


def test_alignment_stops(oracle, gpu_ctx):
    """a start with no inlier (NO_CORRESPONDENCES, 0 iterations), max_iterations = 1 (MAX_ITERATIONS after 1) and a cloud on the base
    frame's z axis (its yaw column is zero: SINGULAR, 0 iterations, with inliers)"""
    import kinematic_icp_b200 as kb
    ko = oracle
    vs = 0.5
    pts = np.random.default_rng(8).uniform(-3, 3, (800, 3))
    om = ko.OracleMap(vs, S.FAR, 20)
    om.add_points(pts)
    gm = _map(kb, gpu_ctx, om)
    try:
        res = align(ko, gm, om, pts[:100], [ko.planar_pose(50.0, 50.0, 0.0)], 0.4, name="no-inlier-start")
        assert res[0]["status"] == AO.NO_CORRESPONDENCES and res[0]["iterations"] == 0
        res = align(ko, gm, om, pts[:100] + 0.01, [ko.IDENTITY], 0.4, max_iterations=1, name="one-iteration")
        assert res[0]["status"] == AO.MAX_ITERATIONS and res[0]["iterations"] == 1
    finally:
        gm.close()
    line = np.stack([np.zeros(40), np.zeros(40), np.linspace(-2.0, 2.0, 40)], 1)
    om = ko.OracleMap(vs, S.FAR, 20)
    om.add_points(line + [0.05, 0.03, 0.0])
    gm = _map(kb, gpu_ctx, om)
    try:
        res = align(ko, gm, om, line, [ko.IDENTITY, ko.planar_pose(0.01, 0.0, 0.3)], 0.4, name="collinear")
        assert all(r["status"] == AO.SINGULAR and r["iterations"] == 0 and r["v"][0] > 0 for r in res)
    finally:
        gm.close()


@pytest.mark.parametrize("cap", [1, 24, 25, 29, 255])
def test_full_voxels(oracle, gpu_ctx, cap):
    """voxels full to `cap` points on a lattice of step 1/8 (many rounds of 32 candidates, exact distance ties) for all three"""
    import kinematic_icp_b200 as kb
    ko = oracle
    rng = np.random.default_rng(cap)
    lattice = np.stack(np.meshgrid(*[np.arange(8) / 8.0] * 3, indexing="ij"), -1).reshape(-1, 3)
    keys = np.array([[i, j, k] for i in range(-1, 2) for j in range(-1, 2) for k in range(-1, 2)], dtype=np.float64)
    pts = np.concatenate([key + lattice[rng.permutation(len(lattice))] for key in keys])
    om = ko.OracleMap(1.0, S.FAR, cap)
    om.add_points(pts)
    assert (om.export_voxels()[1] == cap).all()
    gm = _map(kb, gpu_ctx, om)
    try:
        src = np.concatenate([rng.uniform(-1.5, 1.5, (60, 3)), pts[::97], np.round(rng.uniform(-1, 1, (40, 3)) * 16) / 16])
        pose = ko.planar_pose(0.0625, 0.0, 0.0)
        want = corr(ko, gm, om, src, pose, 0.1, "cap%d" % cap)
        assert 0 < want["n_inliers"] < len(src)
        res = search(ko, gm, om, src, pose, 0.1, (0.125, 0.125, 0.05), (0.0625, 0.0625, 0.05), 2, 5, "cap%d" % cap)
        assert res["kept"][0][1] > 0
        res = align(ko, gm, om, src, [pose, ko.planar_pose(0.03, -0.02, 0.01)], 0.1, max_iterations=4, name="cap%d" % cap)
        assert all(r["v"][0] > 0 for r in res)
    finally:
        gm.close()
