"""The pose search's kernels (k_pose_score, k_pose_select: kinematic-icp_b200/csrc/kicp_pose_search_kernels.cuh) checked without a GPU:
the kernel source compiled by g++ against the SIMT emulator (tests/emu/kps_emu.cpp) and driven by a level loop over the library's
host logic (kicp_pose_search.h), on maps loaded by k_load_voxels or built by AddPoints.  At several launch shapes, on workload and
gate-boundary scenes, ties, an empty map, non-finite points, n = 0 and yaws at +-pi: every returned hypothesis's count exactly, its
sum_sq bit for bit against the oracle restated in the kernel's summation order (tests/pose_search_oracle.py) and within 1e-12 of the
plain sum, its pose bit for bit, the kept set of every level the oracle's, and the same bits at every launch shape."""
import ctypes as C

import numpy as np
import pytest

import gate_scenes as G
import pose_search_oracle as PO
import scenes as S
from emu import harness as H

# (k_pose_score grid, k_pose_select items per CTA): one CTA for every tile and 64 items a CTA (many select passes); a few CTAs
# striding over the tiles; the library's shape (2048 items a CTA)
SHAPES = [(1, 64), (3, 300), (64, 2048)]


def kps_lib():
    L = H.build("kps_emu")
    if not getattr(L, "_typed", False):
        L.km_emu_create.restype = C.c_void_p
        L.km_emu_create.argtypes = [C.c_double, C.c_double, C.c_int32, C.c_uint32]
        L.km_emu_destroy.argtypes = [C.c_void_p]
        L.km_emu_add_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.km_emu_load_voxels.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
        L.kps_emu_search.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.POINTER(PO.Params), C.c_int32, C.c_int32,
                                     C.POINTER(PO.Hypothesis), C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.c_void_p,
                                     C.c_void_p]
        L._typed = True
    return L


class Map:
    def __init__(self, voxel_size, cap, voxels=None, points=None, blocks_cap=60000):
        self.L = kps_lib()
        self.h = C.c_void_p(self.L.km_emu_create(voxel_size, S.FAR, cap, blocks_cap))
        if voxels is not None and len(voxels[1]):
            keys, counts, pts = (np.ascontiguousarray(a, dtype=t) for a, t in zip(voxels, (np.int32, np.int32, np.float64)))
            assert self.L.km_emu_load_voxels(self.h, keys.ctypes.data, counts.ctypes.data, pts.ctypes.data, len(counts)) == 0
        if points is not None:
            p = np.ascontiguousarray(points, dtype=np.float64)
            assert self.L.km_emu_add_points(self.h, p.ctypes.data, len(p), None) == 0

    def search(self, src, prior, tau, half_extent, step, levels, keep, grid, per_cta):
        src = np.ascontiguousarray(src, dtype=np.float64).reshape(-1, 3)
        prior = np.ascontiguousarray(prior, dtype=np.float64)
        p = PO.params(half_extent, step, tau, levels, keep)
        out = (PO.Hypothesis * keep)()
        n_out, n_scored = C.c_int32(), C.c_int64()
        lk = np.full((levels, keep, 3), -7, np.int32)
        ln = np.zeros(levels, np.int32)
        assert self.L.kps_emu_search(self.h, src.ctypes.data if len(src) else None, len(src), prior.ctypes.data, C.byref(p), grid,
                                     per_cta, out, keep, C.byref(n_out), C.byref(n_scored), lk.ctypes.data, ln.ctypes.data) == 0
        return list(out)[: n_out.value], n_scored.value, [[tuple(r) for r in lk[l, : ln[l]]] for l in range(levels)]

    def close(self):
        self.L.km_emu_destroy(self.h)


def check(ko, m, om, src, prior, tau, half_extent, step, levels, keep, name):
    """every launch shape against the oracle's search, and the same bits at every shape"""
    res = PO.search(ko, om, src, prior, tau, half_extent, step, levels, keep)
    first = None
    for grid, per_cta in SHAPES:
        hyps, n_scored, level_kept = m.search(src, prior, tau, half_extent, step, levels, keep, grid, per_cta)
        where = (name, grid, per_cta)
        assert n_scored == res["n_scored"], where
        assert level_kept == res["level_kept"], where
        PO.check_hypotheses(hyps, res, prior, len(src))
        raw = [bytes(h) for h in hyps]
        assert first is None or raw == first, where
        first = raw
    return res


def test_workload_map(oracle, workload):
    """cfg2's map and 400 of its scan points around the prior and around a perturbed prior, three levels"""
    ko = oracle
    w = workload(2)
    m = Map(w.voxel_size, w.max_points_per_voxel, voxels=w.map.export_voxels())
    try:
        src = w.scan[::max(1, len(w.scan) // 400)][:400]
        res = check(ko, m, w.map, src, w.prior, w.tau, (0.2, 0.2, 0.04), (0.1, 0.1, 0.02), 3, 4, "cfg2")
        assert res["kept"][0][1] > 0
        moved = ko.se3_compose(w.prior, ko.planar_pose(0.13, -0.07, 0.015))
        check(ko, m, w.map, src, moved, w.tau, (0.2, 0.2, 0.04), (0.1, 0.1, 0.02), 3, 5, "cfg2-moved")
    finally:
        m.close()


def test_gate_boundary(oracle):
    """The gate scenes of tests/gate_scenes.py (map points at prev(tau), tau and next(tau) from the prior's queries, on voxel faces,
    edges and corners; the exact (3, 4, 12) 2^k cases): the prior's own hypothesis and its neighbours on a fine lattice."""
    ko = oracle
    for sc in G.gate_scenes(ko):
        m = Map(sc.voxel_size, sc.cap, voxels=sc.voxels)
        try:
            src = np.asarray(sc.scan, dtype=np.float64)[:150]
            prior = ko.se3_compose(sc.last, sc.odom)
            check(ko, m, sc.om, src, prior, sc.tau, (1e-9, 1e-9, 1e-9), (1e-9, 1e-9, 1e-9), 2, 3, sc.name)
        finally:
            m.close()


def test_ties(oracle):
    """Exact and ulp-level near ties between voxels and inside one voxel (tests/scenes.py), and exact score ties between hypotheses
    (a map of one repeated pattern), broken by the rest of the key"""
    ko = oracle
    for sc in S.tie_scenes(ko):
        m = Map(sc.voxel_size, sc.cap, voxels=sc.voxels)
        try:
            src = np.asarray(sc.scan, dtype=np.float64)[:120]
            check(ko, m, sc.om, src, ko.se3_compose(sc.last, sc.odom), sc.tau, (0.25, 0.25, 0.0), (0.125, 0.125, 0.1), 2, 6, sc.name)
        finally:
            m.close()
    vs = 1.0
    grid = np.stack(np.meshgrid(np.arange(-4, 5), np.arange(-4, 5), [0.0], indexing="ij"), -1).reshape(-1, 3) + 0.5
    om = ko.OracleMap(vs, S.FAR, 20)
    om.add_points(grid)
    m = Map(vs, 20, points=grid)
    try:
        res = check(ko, m, om, grid[20:40], ko.IDENTITY, 0.3, (2.0, 2.0, 0.0), (1.0, 1.0, 0.1), 1, 8, "lattice-ties")
        assert len({(c, s) for _, c, s, _ in res["kept"]}) < len(res["kept"])  # the rest of the key decided
    finally:
        m.close()


def test_empty_map_nonfinite_n0_and_yaw_pi(oracle):
    """An empty map (every score (0, 0): the keep points nearest the prior by the key), non-finite source points, n = 0, and a
    level 0 whose yaws reach +-pi"""
    ko = oracle
    vs = 0.5
    rng = np.random.default_rng(8)
    src = S.with_nonfinite(rng.uniform(-3, 3, (200, 3)), vs)
    m = Map(vs, 20)
    try:
        res = check(ko, m, ko.OracleMap(vs, S.FAR, 20), src, ko.IDENTITY, 1.0, (0.2, 0.2, 0.2), (0.1, 0.1, 0.1), 2, 7, "empty")
        assert [L for L, *_ in res["kept"]][:3] == [(0, 0, 0), (-1, 0, 0), (0, -1, 0)]
    finally:
        m.close()
    pts = rng.uniform(-3, 3, (800, 3))
    om = ko.OracleMap(vs, S.FAR, 20)
    om.add_points(pts)
    m = Map(vs, 20, points=pts)
    try:
        res = check(ko, m, om, src, ko.planar_pose(0.1, 0.05, 0.02), 0.4, (0.1, 0.1, 0.05), (0.05, 0.05, 0.05), 2, 4, "nonfinite")
        assert res["kept"][0][1] > 0
        check(ko, m, om, np.zeros((0, 3)), ko.IDENTITY, 0.4, (0.1, 0.1, 0.1), (0.1, 0.1, 0.1), 2, 4, "n0")
        check(ko, m, om, pts[:60], ko.planar_pose(0.0, 0.0, 3.0), 0.4, (0.0, 0.0, np.pi), (0.1, 0.1, np.pi / 4), 2, 5, "yaw-pi")
    finally:
        m.close()
