"""The planar alignment's kernels (k_align_eval, k_align_step, k_align_finish: kinematic-icp_b200/csrc/kicp_align_kernels.cuh) checked
without a GPU: the kernel source compiled by g++ against the SIMT emulator (tests/emu/kal_emu.cpp) and driven by the library's launch
sequence restated there, on maps loaded by k_load_voxels or built by AddPoints.  At three k_align_eval grids (one CTA, three CTAs
striding over the alignments' slots, one CTA per slot), on workload and gate-boundary scenes, ties, an empty map, n = 0, non-finite
points, a start without inliers, a collinear cloud, max_iterations = 1 and yaws at +-pi: every iteration's pose and status, the
iteration count and the report at the returned pose bit for bit against the oracle's restatement (tests/align_planar_oracle.py), the
same bits at every grid and on a second run, and a call of many starts equal to one call per start."""
import ctypes as C
import math

import numpy as np

import align_planar_oracle as AO
import gate_scenes as G
import scenes as S
from emu import harness as H


def kal_lib():
    L = H.build("kal_emu")
    if not getattr(L, "_typed", False):
        L.km_emu_create.restype = C.c_void_p
        L.km_emu_create.argtypes = [C.c_double, C.c_double, C.c_int32, C.c_uint32]
        L.km_emu_destroy.argtypes = [C.c_void_p]
        L.km_emu_add_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.km_emu_load_voxels.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
        L.kal_emu_align.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.POINTER(AO.Params), C.c_int32,
                                    C.POINTER(AO.Alignment), C.c_void_p, C.c_void_p]
        L._typed = True
    return L


class Map:
    def __init__(self, voxel_size, cap, voxels=None, points=None, blocks_cap=60000):
        self.L = kal_lib()
        self.h = C.c_void_p(self.L.km_emu_create(voxel_size, S.FAR, cap, blocks_cap))
        if voxels is not None and len(voxels[1]):
            keys, counts, pts = (np.ascontiguousarray(a, dtype=t) for a, t in zip(voxels, (np.int32, np.int32, np.float64)))
            assert self.L.km_emu_load_voxels(self.h, keys.ctypes.data, counts.ctypes.data, pts.ctypes.data, len(counts)) == 0
        if points is not None:
            p = np.ascontiguousarray(points, dtype=np.float64)
            assert self.L.km_emu_add_points(self.h, p.ctypes.data, len(p), None) == 0

    def align(self, src, starts, tau, max_iterations, convergence, grid):
        src = np.ascontiguousarray(src, dtype=np.float64).reshape(-1, 3)
        starts = np.ascontiguousarray(starts, dtype=np.float64).reshape(-1, 7)
        k = len(starts)
        p = AO.Params(tau, convergence, max_iterations)
        out = (AO.Alignment * k)()
        traj = np.full((k, max_iterations, 7), np.nan)
        st = np.full((k, max_iterations), -1, np.int32)
        assert self.L.kal_emu_align(self.h, src.ctypes.data if len(src) else None, len(src), starts.ctypes.data, k, C.byref(p), grid, out,
                                    traj.ctypes.data, st.ctypes.data) == 0
        return list(out), traj, st

    def close(self):
        self.L.km_emu_destroy(self.h)


def grids(n, k):
    """one CTA; three (fewer than the alignments' slots: blocks grid-stride); one CTA per slot"""
    return [1, 3, k * AO.slots(n)]


def check(ko, m, om, src, starts, tau, max_iterations=10, convergence=1e-3, name=""):
    """every grid against the oracle (trajectory, status, iterations, report), the same bits at every grid and on a second run"""
    starts = np.asarray(starts, dtype=np.float64).reshape(-1, 7)
    want = [AO.align(ko, om, src, T0, tau, max_iterations, convergence) for T0 in starts]
    first = None
    for g in grids(len(np.asarray(src).reshape(-1, 3)), len(starts)):
        out, traj, st = m.align(src, starts, tau, max_iterations, convergence, g)
        for a, (o, res) in enumerate(zip(out, want)):
            where = (name, g, a)
            AO.check_alignment(o, res, where)
            assert np.array_equal(traj[a], np.array(res["traj"])), where
            assert list(st[a]) == res["statuses"], where
        raw = [bytes(o) for o in out]
        assert first is None or raw == first, (name, g)
        first = raw
    out, _, _ = m.align(src, starts, tau, max_iterations, convergence, 3)
    assert [bytes(o) for o in out] == first, (name, "second run")
    return want


def test_workload_map(oracle, workload):
    """cfg2's map and 600 of its scan points (three slots), from the prior and from a planar offset of the true pose, gate 0.3 m: one
    start converges, the other runs out of iterations"""
    ko = oracle
    w = workload(2)
    m = Map(w.voxel_size, w.max_points_per_voxel, voxels=w.map.export_voxels())
    try:
        src = w.scan[:: max(1, len(w.scan) // 600)][:600]
        starts = [w.prior, ko.se3_compose(w.true_pose, ko.planar_pose(0.13, -0.07, 0.015))]
        res = check(ko, m, w.map, src, starts, 0.3, name="cfg2")
        assert [r["status"] for r in res] == [AO.CONVERGED, AO.MAX_ITERATIONS] and all(r["v"][0] > 0 for r in res)
    finally:
        m.close()


def test_batched_equals_one_by_one(oracle, workload):
    """64 starts in one call == each start alone (the alignment's bits do not depend on the others)"""
    ko = oracle
    w = workload(2)
    m = Map(w.voxel_size, w.max_points_per_voxel, voxels=w.map.export_voxels())
    try:
        src = w.scan[:: max(1, len(w.scan) // 300)][:300]
        rng = np.random.default_rng(11)
        starts = np.array([ko.se3_compose(w.true_pose, ko.planar_pose(*rng.uniform([-0.2, -0.2, -0.05], [0.2, 0.2, 0.05])))
                           for _ in range(64)])
        many, traj, _ = m.align(src, starts, 0.3, 3, 1e-3, 40)
        for a in (0, 17, 63):
            one, t1, _ = m.align(src, starts[a], 0.3, 3, 1e-3, 2)
            assert bytes(one[0]) == bytes(many[a]) and np.array_equal(t1[0], traj[a]), a
        for a in (5, 40):
            AO.check_alignment(many[a], AO.align(ko, w.map, src, starts[a], 0.3, 3, 1e-3), a)
    finally:
        m.close()


def test_gate_boundary(oracle):
    """the gate scenes of tests/gate_scenes.py (map points at prev(tau), tau and next(tau) from the prior's queries, on voxel faces,
    edges and corners), aligned from the prior"""
    ko = oracle
    for sc in G.gate_scenes(ko):
        m = Map(sc.voxel_size, sc.cap, voxels=sc.voxels)
        try:
            src = np.asarray(sc.scan, dtype=np.float64)[:150]
            check(ko, m, sc.om, src, [ko.se3_compose(sc.last, sc.odom)], sc.tau, max_iterations=3, name=sc.name)
        finally:
            m.close()


def test_ties(oracle):
    """exact and ulp-level near ties between voxels and inside one voxel (tests/scenes.py)"""
    ko = oracle
    for sc in S.tie_scenes(ko):
        m = Map(sc.voxel_size, sc.cap, voxels=sc.voxels)
        try:
            src = np.asarray(sc.scan, dtype=np.float64)[:120]
            check(ko, m, sc.om, src, [ko.se3_compose(sc.last, sc.odom)], sc.tau, max_iterations=3, name=sc.name)
        finally:
            m.close()


def test_edges(oracle):
    """an empty map and n = 0 (NO_CORRESPONDENCES after 0 iterations at the start's bits), non-finite points, a start with no inlier,
    a cloud on the base frame's z axis (its yaw column is zero: SINGULAR), max_iterations = 1 (MAX_ITERATIONS) and starts at yaw +-pi"""
    ko = oracle
    vs = 0.5
    rng = np.random.default_rng(8)
    pts = rng.uniform(-3, 3, (800, 3))
    start = ko.planar_pose(0.1, 0.05, 0.02)
    m = Map(vs, 20)
    try:
        res = check(ko, m, ko.OracleMap(vs, S.FAR, 20), pts[:100], [start], 0.4, name="empty-map")
        assert res[0]["status"] == AO.NO_CORRESPONDENCES and res[0]["iterations"] == 0 and res[0]["pose"] == list(start)
    finally:
        m.close()
    om = ko.OracleMap(vs, S.FAR, 20)
    om.add_points(pts)
    m = Map(vs, 20, points=pts)
    try:
        res = check(ko, m, om, np.zeros((0, 3)), [start], 0.4, name="n0")
        assert res[0]["status"] == AO.NO_CORRESPONDENCES and res[0]["iterations"] == 0 and res[0]["pose"] == list(start)
        src = S.with_nonfinite(pts[:200] + rng.normal(0, 0.02, (200, 3)), vs)
        res = check(ko, m, om, src, [start, ko.IDENTITY], 0.4, name="nonfinite")
        assert all(r["v"][0] > 0 for r in res)
        res = check(ko, m, om, pts[:100], [ko.planar_pose(50.0, 50.0, 0.0)], 0.4, name="no-inlier-start")
        assert res[0]["status"] == AO.NO_CORRESPONDENCES and res[0]["iterations"] == 0
        res = check(ko, m, om, pts[:100] + 0.01, [ko.IDENTITY], 0.4, max_iterations=1, name="one-iteration")
        assert res[0]["status"] == AO.MAX_ITERATIONS and res[0]["iterations"] == 1
        res = check(ko, m, om, pts[:120], [ko.planar_pose(0.02, 0.0, math.pi), ko.planar_pose(0.0, 0.01, -math.pi),
                                           ko.planar_pose(0.0, 0.0, math.pi - 1e-3)], 0.4, max_iterations=4, name="yaw-pi")
        assert all(r["v"][0] > 0 for r in res)
    finally:
        m.close()
    line = np.stack([np.zeros(40), np.zeros(40), np.linspace(-2.0, 2.0, 40)], 1)  # collinear along the base frame's z axis
    om = ko.OracleMap(vs, S.FAR, 20)
    om.add_points(line + [0.05, 0.03, 0.0])
    m = Map(vs, 20, points=line + [0.05, 0.03, 0.0])
    try:
        res = check(ko, m, om, line, [ko.IDENTITY, ko.planar_pose(0.01, 0.0, 0.3)], 0.4, name="collinear")
        assert all(r["status"] == AO.SINGULAR and r["iterations"] == 0 and r["v"][0] > 0 for r in res)
    finally:
        m.close()
