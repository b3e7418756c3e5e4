"""Free-space clearing under the SIMT emulator (tests/emu/kfree_emu.cpp: kicp_free_space_kernels.cuh with the launch sequences of
kicp_map.cu on the emulated map of km_emu / kpm_emu) against the oracle of tests/free_space_oracle.py: the synchronous sequence exactly
(exports byte for byte, statistics), independent of the launch shape, with and without a frozen prior; the frame path's sequence
against the option-off frame followed by the oracle; and a result block that is not KICP_OK leaving the map bit-identical."""
import ctypes as C

import numpy as np
import pytest

import free_space_oracle as F
from emu import harness as H

VS, MD = 0.5, 30.0
STAT_KEYS = ("rays", "visits", "cleared_voxels", "cleared_points", "prior_contradicted")


def _lib():
    L = H.build("kfree_emu")
    L.km_emu_create.restype = C.c_void_p
    L.km_emu_create.argtypes = [C.c_double, C.c_double, C.c_int32, C.c_uint32]
    L.km_emu_destroy.argtypes = [C.c_void_p]
    for f in (L.km_emu_num_points, L.km_emu_num_voxels):
        f.restype, f.argtypes = C.c_int64, [C.c_void_p]
    L.km_emu_export.restype = C.c_int64
    L.km_emu_export.argtypes = [C.c_void_p] * 4
    L.km_emu_load_voxels.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    for f in (L.kpm_emu_freeze, L.kpm_emu_thaw):
        f.argtypes = [C.c_void_p]
    L.kpm_emu_prior_blocks.restype = C.c_uint32
    L.kpm_emu_prior_blocks.argtypes = [C.c_void_p]
    L.kpm_emu_add_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    L.kpm_emu_update_pose_async.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32]
    L.kpm_emu_table.restype = C.c_int64
    L.kpm_emu_table.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]
    L.kfree_emu_clear.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_double, C.c_int32, C.c_int32, C.c_void_p]
    L.kfree_emu_update_pose_async.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_double,
                                              C.c_int32, C.c_int32, C.c_void_p]
    return L


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class _Map:
    def __init__(self, L, voxels=None, freeze=False, live_points=None):
        self.L = L
        self.h = C.c_void_p(L.km_emu_create(VS, MD, 20, 60000))
        if voxels is not None:
            keys, counts = np.ascontiguousarray(voxels[0], np.int32), np.ascontiguousarray(voxels[1], np.int32)
            pts = _f64(voxels[2])
            assert L.km_emu_load_voxels(self.h, keys.ctypes.data, counts.ctypes.data, pts.ctypes.data, len(counts)) == 0
        if freeze:
            L.kpm_emu_freeze(self.h)
        if live_points is not None:
            p = _f64(live_points)
            assert L.kpm_emu_add_points(self.h, p.ctypes.data, len(p), None) == 0

    def P(self):
        return int(self.L.kpm_emu_prior_blocks(self.h))

    def export(self):
        nv, npts = self.L.km_emu_num_voxels(self.h), self.L.km_emu_num_points(self.h)
        keys, counts, pts = np.zeros((nv, 3), np.int32), np.zeros(nv, np.int32), np.zeros((npts, 3))
        assert self.L.km_emu_export(self.h, keys.ctypes.data, counts.ctypes.data, pts.ctypes.data) == nv
        return keys, counts, pts

    def clear(self, pts, pose, origin, margin, min_misses, grid=0):
        pts, pose, origin = _f64(pts), _f64(pose), _f64(origin)
        st = np.zeros(5, np.int64)
        assert self.L.kfree_emu_clear(self.h, pts.ctypes.data, len(pts), pose.ctypes.data, origin.ctypes.data, margin, min_misses, grid,
                                      st.ctypes.data) == 0
        return dict(zip(STAT_KEYS, st.tolist()))

    def frame(self, pts, n_actual, pose, status, origin=None, margin=0.0, min_misses=0, grid=0):
        pts, pose = _f64(pts), _f64(pose)
        if not min_misses:
            assert self.L.kpm_emu_update_pose_async(self.h, pts.ctypes.data, len(pts), n_actual, pose.ctypes.data, status) == 0
            return None
        origin = _f64(origin)
        st = np.zeros(5, np.int64)
        assert self.L.kfree_emu_update_pose_async(self.h, pts.ctypes.data, len(pts), n_actual, pose.ctypes.data, status, origin.ctypes.data,
                                                  margin, min_misses, grid, st.ctypes.data) == 0
        return dict(zip(STAT_KEYS, st.tolist()))

    def tables_agree(self):
        out = [np.zeros((1 << 20, 4), np.int32) for _ in range(2)]
        n = [self.L.kpm_emu_table(self.h, f, out[f].ctypes.data, len(out[f])) for f in (0, 1)]
        return sorted(map(tuple, out[0][:n[0]].tolist())) == sorted(map(tuple, out[1][:n[1]].tolist()))

    def close(self):
        self.L.kpm_emu_thaw(self.h)
        self.L.km_emu_destroy(self.h)


def _bytes(v):
    return tuple(np.ascontiguousarray(a).tobytes() for a in v)


def _sorted(voxels):
    keys, counts, pts = voxels
    starts = np.r_[0, np.cumsum(counts)[:-1]].astype(np.int64)
    order = np.lexsort(np.asarray(keys).T[::-1])
    return [(tuple(keys[v]), pts[starts[v]:starts[v] + counts[v]].tobytes()) for v in order]


def _scene(seed):
    """a wall at x ~ 12 m, a 'van' of live voxels in front of it, clutter around; rays from near the origin to the wall"""
    rng = np.random.default_rng(seed)
    wall = np.c_[np.full(1500, 12.2) + rng.uniform(0, 0.2, 1500), rng.uniform(-6, 6, 1500), rng.uniform(-1, 2, 1500)]
    van = np.c_[rng.uniform(5, 7, 800), rng.uniform(-1.5, 1.5, 800), rng.uniform(-0.5, 1.5, 800)]
    clutter = rng.uniform(-10, 10, (600, 3))
    rays = np.c_[np.full(900, 12.3) + rng.uniform(0, 0.05, 900), rng.uniform(-5, 5, 900), rng.uniform(-0.8, 1.8, 900)]
    return np.round(wall * 1024) / 1024, np.round(van * 1024) / 1024, np.round(clutter * 1024) / 1024, np.round(rays * 1024) / 1024


POSE = np.array([0.0, 0.0, np.sin(0.05), np.cos(0.05), 0.4, -0.3, 0.1])


@pytest.mark.parametrize("prior", [False, True])
def test_synchronous_sequence_matches_the_oracle(oracle, prior):
    L = _lib()
    wall, van, clutter, rays = _scene(1)
    base = _Map(L, live_points=np.concatenate([wall, clutter]))
    voxels = base.export()
    base.close()
    m = _Map(L, voxels, freeze=prior, live_points=van)
    try:
        before = m.export()
        P = m.P()
        for margin, mm in ((0.0, 1), (0.5, 2), (0.25, 3)):
            want, wst = F.clear_free_space(oracle, before, P, VS, MD, rays, POSE, [0.1, 0.0, 0.3], margin, mm)
            got_st = m.clear(rays, POSE, [0.1, 0.0, 0.3], margin, mm, grid=0)
            assert got_st == wst, (margin, mm)
            got = m.export()
            assert _bytes(got) == _bytes(want), (margin, mm)
            assert m.tables_agree()
            assert _bytes(got[:2]) and int(got[1][:P].sum()) == int(before[1][:P].sum())
            before = got
        assert wst["rays"] == len(rays)
    finally:
        m.close()


def test_van_is_cleared_live_and_counted_as_prior(oracle):
    L = _lib()
    wall, van, clutter, rays = _scene(2)
    for prior in (False, True):
        base = _Map(L, live_points=np.concatenate([wall, van]))
        voxels = base.export()
        base.close()
        m = _Map(L, voxels, freeze=prior)
        try:
            st = m.clear(rays, np.array([0, 0, 0, 1.0, 0, 0, 0]), [0.0, 0.0, 0.5], 0.5, 2)
            want, wst = F.clear_free_space(oracle, voxels, len(voxels[1]) if prior else 0, VS, MD, rays, [0, 0, 0, 1.0, 0, 0, 0],
                                           [0.0, 0.0, 0.5], 0.5, 2)
            assert st == wst and _bytes(m.export()) == _bytes(want)
            if prior:
                assert st["cleared_voxels"] == 0 and st["prior_contradicted"] > 0
            else:
                assert st["cleared_voxels"] > 0 and st["prior_contradicted"] == 0
        finally:
            m.close()


def test_launch_shape_does_not_change_the_result(oracle):
    L = _lib()
    wall, van, clutter, rays = _scene(3)
    voxels = None
    base = _Map(L, live_points=np.concatenate([wall, van, clutter]))
    voxels = base.export()
    base.close()
    res = []
    for grid in (1, 2, 0):
        m = _Map(L, voxels)
        try:
            st = m.clear(rays, POSE, [0.0, 0.0, 0.5], 0.25, 2, grid=grid)
            res.append((st, _bytes(m.export())))
        finally:
            m.close()
    assert res[0] == res[1] == res[2]


@pytest.mark.parametrize("prior", [False, True])
def test_frame_path_sequence_equals_option_off_then_clearing(oracle, prior):
    L = _lib()
    wall, van, clutter, rays = _scene(4)
    base = _Map(L, live_points=np.concatenate([wall, clutter]))
    voxels = base.export()
    base.close()
    frame = np.concatenate([rays, wall[:300]])
    n_actual = len(frame) - 17
    origin = [0.2, 0.0, 0.4]
    a, b = _Map(L, voxels, freeze=prior, live_points=van), _Map(L, voxels, freeze=prior, live_points=van)
    try:
        st = a.frame(frame, n_actual, POSE, 0, origin, 0.5, 2)
        b.frame(frame, n_actual, POSE, 0)
        want, wst = F.clear_free_space(oracle, b.export(), b.P(), VS, MD, frame[:n_actual], POSE, origin, 0.5, 2)
        assert st == wst
        assert wst["cleared_voxels"] + wst["prior_contradicted"] > 0
        got = a.export()
        assert _sorted(got) == _sorted(want)
        P = a.P()
        assert _bytes((got[0][:P], got[1][:P])) == _bytes((want[0][:P], want[1][:P]))
        assert a.tables_agree()
    finally:
        a.close()
        b.close()


def test_frame_path_leaves_the_map_bit_identical_on_a_failed_result(oracle):
    L = _lib()
    wall, van, clutter, rays = _scene(5)
    m = _Map(L, live_points=np.concatenate([wall, van]))
    try:
        before = m.export()
        st = m.frame(rays, len(rays), POSE, 3, [0.0, 0.0, 0.0], 0.0, 1)
        assert st == dict.fromkeys(STAT_KEYS, 0)
        assert _bytes(m.export()) == _bytes(before)
        assert m.tables_agree()
    finally:
        m.close()
