"""The correspondence report's kernels (k_corr_eval, k_corr_finish: kinematic-icp_b200/csrc/kicp_corr_kernels.cuh) checked without a
GPU: the kernel source compiled by g++ against the SIMT emulator (tests/emu/kc_emu.cpp) on maps loaded by k_load_voxels or built by
AddPoints, at several launch shapes, with the source count read from a device word and the pose from a result block.  Per-point
neighbours, distances and the inlier mask bit for bit, the counts exactly and the sums to 1e-12 against the oracle's composition
(tests/corr_oracle.py); the sums' bits the same from run to run."""
import ctypes as C

import numpy as np
import pytest

import gate_scenes as G
import scenes as S
from corr_oracle import CorrStats, check_stats, oracle_corr
from emu import harness as H

DBL_MAX = np.finfo(np.float64).max


def kc_lib():
    L = H.build("kc_emu")
    if not getattr(L, "_typed", False):
        L.km_emu_create.restype = C.c_void_p
        L.km_emu_create.argtypes = [C.c_double, C.c_double, C.c_int32, C.c_uint32]
        L.km_emu_destroy.argtypes = [C.c_void_p]
        L.km_emu_add_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.km_emu_load_voxels.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
        L.kc_emu_correspondences.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_double,
                                             C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L._typed = True
    return L


class Map:
    def __init__(self, voxel_size, cap, voxels=None, points=None, blocks_cap=60000):
        self.L = kc_lib()
        self.h = C.c_void_p(self.L.km_emu_create(voxel_size, S.FAR, cap, blocks_cap))
        if voxels is not None and len(voxels[1]):
            keys, counts, pts = (np.ascontiguousarray(a, dtype=t) for a, t in zip(voxels, (np.int32, np.int32, np.float64)))
            assert self.L.km_emu_load_voxels(self.h, keys.ctypes.data, counts.ctypes.data, pts.ctypes.data, len(counts)) == 0
        if points is not None:
            p = np.ascontiguousarray(points, dtype=np.float64)
            assert self.L.km_emu_add_points(self.h, p.ctypes.data, len(p), None) == 0

    def corr(self, src, pose, tau, grid, threads, n_dev=-1, from_result=False, status=0):
        """k_corr_eval over the buffer src (n_dev >= 0: the count read from a device word), then k_corr_finish"""
        src = np.ascontiguousarray(src, dtype=np.float64).reshape(-1, 3)
        pose = np.ascontiguousarray(pose, dtype=np.float64)
        n = len(src)
        pts, dist, inl = np.full((n, 3), -7.0), np.full(n, -7.0), np.full(n, 7, np.uint8)  # every row below the count must be written
        parts = np.full((grid, 8), np.nan)
        st = CorrStats()
        assert self.L.kc_emu_correspondences(self.h, src.ctypes.data if n else None, n, n_dev, pose.ctypes.data, int(from_result), status,
                                             tau, grid, threads, pts.ctypes.data, dist.ctypes.data, inl.ctypes.data, parts.ctypes.data,
                                             C.addressof(st)) == 0
        return pts, dist, inl, st, parts

    def close(self):
        self.L.km_emu_destroy(self.h)


def shapes(n):
    """one warp in all; fewer warps than points; the library's 256-thread CTAs, more warps than points"""
    return [(1, 32), (3, 64), ((n + 7) // 8 + 3, 256)]


def check(ko, m, om, src, pose, tau, name, status=0):
    """every shape, with the count on the host and from a device word (the buffer then holds 5 more rows than the count), the pose
    as an argument and from a result block"""
    po, do, io, want = oracle_corr(ko, om, src, pose, tau)
    n = len(src)
    padded = np.concatenate([np.asarray(src, dtype=np.float64).reshape(-1, 3), np.full((5, 3), 1.0)])
    for grid, threads in shapes(n):
        for dev in (False, True):
            if dev:
                pe, de, ie, st, _ = m.corr(padded, pose, tau, grid, threads, n_dev=n, from_result=True, status=status)
                assert (de[n:] == -7.0).all() and (ie[n:] == 7).all(), (name, "rows beyond the device count were written")
                pe, de, ie = pe[:n], de[:n], ie[:n]
            else:
                pe, de, ie, st, _ = m.corr(src, pose, tau, grid, threads)
            where = (name, grid, threads, dev)
            assert S.same_bits(de, do) and S.same_bits(pe, po), where
            assert np.array_equal(ie.astype(bool), io) and set(np.unique(ie)) <= {0, 1}, where
            check_stats(st, want)
    return want


def test_workload_map(oracle, workload):
    """cfg2's map, its scan at the prior and at a perturbed pose, with uniform far points (empty neighbourhoods)."""
    ko = oracle
    w = workload(2)
    m = Map(w.voxel_size, w.max_points_per_voxel, voxels=w.map.export_voxels())
    try:
        rng = np.random.default_rng(4)
        src = np.concatenate([w.scan[:1200], rng.uniform(-150, 150, (200, 3))])
        want = check(ko, m, w.map, src, w.prior, w.tau, "cfg2")
        assert 0 < want["n_inliers"] < len(src)
        check(ko, m, w.map, src[:500], ko.se3_compose(w.prior, ko.planar_pose(0.3, -0.2, 0.05)), 2.0 * w.tau, "cfg2-moved")
    finally:
        m.close()


def test_gate_boundary(oracle):
    """The gate scenes of tests/gate_scenes.py: every point alone with one map point at a reference norm of prev(tau), tau or
    next(tau), and the exact (3, 4, 12) 2^k cases.  The inlier count is the reference's count of norms below tau."""
    ko = oracle
    for sc in G.gate_scenes(ko):
        m = Map(sc.voxel_size, sc.cap, voxels=sc.voxels)
        try:
            src = np.asarray(sc.scan, dtype=np.float64)
            want = check(ko, m, sc.om, src, ko.se3_compose(sc.last, sc.odom), sc.tau, sc.name)
            assert want["n_inliers"] == sc.expected_n, sc.name
        finally:
            m.close()


def test_ties(oracle):
    """Exact and ulp-level near ties between voxels and inside one voxel (tests/scenes.py)."""
    ko = oracle
    for sc in S.tie_scenes(ko):
        m = Map(sc.voxel_size, sc.cap, voxels=sc.voxels)
        try:
            check(ko, m, sc.om, np.asarray(sc.scan, dtype=np.float64)[:500], ko.se3_compose(sc.last, sc.odom), sc.tau, sc.name)
        finally:
            m.close()


def test_empty_map_nonfinite_points_and_nan_pose(oracle):
    """An empty map (nothing found, no inliers, fitness 0); non-finite source points; a NaN pose as a frame with
    KICP_WARN_NO_CORRESPONDENCES leaves it in its result block (every distance DBL_MAX, no inliers); n = 0."""
    ko = oracle
    vs = 0.5
    rng = np.random.default_rng(8)
    src = S.with_nonfinite(rng.uniform(-3, 3, (300, 3)), vs)
    om_empty = ko.OracleMap(vs, S.FAR, 20)
    m = Map(vs, 20)
    try:
        want = check(ko, m, om_empty, src, ko.IDENTITY, 1.0, "empty")
        assert want["n_inliers"] == 0
    finally:
        m.close()
    pts = rng.uniform(-3, 3, (800, 3))
    om = ko.OracleMap(vs, S.FAR, 20)
    om.add_points(pts)
    m = Map(vs, 20, points=pts)
    try:
        want = check(ko, m, om, src, ko.planar_pose(0.1, 0.05, 0.02), 0.4, "nonfinite")
        assert 0 < want["n_inliers"] < len(src)
        nan_pose = np.full(7, np.nan)
        want = check(ko, m, om, src, nan_pose, 0.4, "nan-pose", status=16)
        assert want["n_inliers"] == 0
        _, d, inl, st, _ = m.corr(src, nan_pose, 0.4, 4, 256, n_dev=len(src), from_result=True, status=16)
        assert (d == DBL_MAX).all() and not inl.any() and st.n_inliers == 0 and st.fitness == 0.0
        check(ko, m, om, np.zeros((0, 3)), ko.IDENTITY, 0.4, "n0")
    finally:
        m.close()


@pytest.mark.parametrize("cap", [1, 33, 255])
def test_full_voxels(oracle, cap):
    """Voxels of up to 255 points on a lattice of step 1/8 (many rounds of 32 candidates, exact distance ties)."""
    ko = oracle
    vs = 1.0
    rng = np.random.default_rng(cap)
    lattice = np.stack(np.meshgrid(*[np.arange(8) / 8.0] * 3, indexing="ij"), -1).reshape(-1, 3)
    keys = np.array([[i, j, k] for i in range(-1, 2) for j in range(-1, 2) for k in range(-1, 2)], dtype=np.float64)
    pts = np.concatenate([key + lattice[rng.permutation(len(lattice))] for key in keys])
    om = ko.OracleMap(vs, S.FAR, cap)
    om.add_points(pts)
    m = Map(vs, cap, points=pts)
    try:
        src = np.concatenate([rng.uniform(-1.5, 1.5, (60, 3)), pts[::97], np.round(rng.uniform(-1, 1, (40, 3)) * 16) / 16])
        want = check(ko, m, om, src, ko.planar_pose(0.0625, 0.0, 0.0), 0.1, "cap%d" % cap)
        assert 0 < want["n_inliers"] < len(src)
    finally:
        m.close()


def test_same_bits_from_run_to_run(oracle, workload):
    """Two runs at one launch shape give the same per-CTA partials and the same statistics, bit for bit (no atomics)."""
    w = workload(2)
    m = Map(w.voxel_size, w.max_points_per_voxel, voxels=w.map.export_voxels())
    try:
        src = w.scan[:1500]
        runs = [m.corr(src, w.prior, w.tau, 7, 256, n_dev=len(src), from_result=True) for _ in range(2)]
        (_, _, _, s1, p1), (_, _, _, s2, p2) = runs
        assert S.same_bits(p1, p2)
        assert bytes(s1) == bytes(s2) and s1.n_inliers > 0
    finally:
        m.close()
