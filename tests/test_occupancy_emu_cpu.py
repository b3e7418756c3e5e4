"""Occupancy evidence under the SIMT emulator (tests/emu/kocc_emu.cpp: the changed kernels with kicp_map.cu's launch sequences on the
emulated map of km_emu / kpm_emu) against tests/occupancy_oracle.py: sequences of clearing calls interleaved with inserts, evictions,
freeze / thaw, a new set call and a load match the oracle byte for byte in exports, evidence and statistics at several launch shapes;
the frame path's sequence equals the option-off frame followed by the oracle; and a result block that is not KICP_OK leaves the map and
its evidence bit-identical."""
import ctypes as C

import numpy as np
import pytest

import occupancy_oracle as O
from emu import harness as H

VS, MD = 0.5, 30.0
STAT_KEYS = ("rays", "visits", "cleared_voxels", "cleared_points", "prior_contradicted")
POSE = np.array([0.0, 0.0, np.sin(0.05), np.cos(0.05), 0.4, -0.3, 0.1])
ORIGIN = [0.1, 0.0, 0.3]


def _lib():
    L = H.build("kocc_emu")
    L.km_emu_create.restype = C.c_void_p
    L.km_emu_create.argtypes = [C.c_double, C.c_double, C.c_int32, C.c_uint32]
    L.km_emu_destroy.argtypes = [C.c_void_p]
    for f in (L.km_emu_num_points, L.km_emu_num_voxels):
        f.restype, f.argtypes = C.c_int64, [C.c_void_p]
    L.km_emu_export.restype = C.c_int64
    L.km_emu_export.argtypes = [C.c_void_p] * 4
    for f in (L.kocc_emu_freeze, L.kpm_emu_thaw):
        f.argtypes = [C.c_void_p]
    L.kpm_emu_prior_blocks.restype = C.c_uint32
    L.kpm_emu_prior_blocks.argtypes = [C.c_void_p]
    L.kpm_emu_spare_mirrors_prior.argtypes = [C.c_void_p]
    L.kocc_emu_spare_mirrors_prior.argtypes = [C.c_void_p]
    L.kpm_emu_table.restype = C.c_int64
    L.kpm_emu_table.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]
    L.kocc_emu_set.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    L.kocc_emu_evidence.restype = C.c_int64
    L.kocc_emu_evidence.argtypes = [C.c_void_p, C.c_void_p]
    L.kocc_emu_load.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    L.kocc_emu_add_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    L.kocc_emu_remove_far.argtypes = [C.c_void_p, C.c_void_p]
    L.kocc_emu_clear.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_double, C.c_int32, C.c_int32, C.c_void_p]
    L.kocc_emu_update_pose_async.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_double,
                                             C.c_int32, C.c_int32, C.c_void_p]
    return L


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _bytes(v):
    return tuple(np.ascontiguousarray(a).tobytes() for a in v)


class _Map:
    def __init__(self, L, grid=0):
        self.L, self.grid = L, grid
        self.h = C.c_void_p(L.km_emu_create(VS, MD, 20, 60000))

    def set(self, occ):
        self.L.kocc_emu_set(self.h, *(occ if occ else (0, 0, 0, 0)))

    def P(self):
        return int(self.L.kpm_emu_prior_blocks(self.h))

    def export(self):
        nv, npts = self.L.km_emu_num_voxels(self.h), self.L.km_emu_num_points(self.h)
        keys, counts, pts = np.zeros((nv, 3), np.int32), np.zeros(nv, np.int32), np.zeros((npts, 3))
        assert self.L.km_emu_export(self.h, keys.ctypes.data, counts.ctypes.data, pts.ctypes.data) == nv
        return keys, counts, pts

    def evidence(self):
        out = np.zeros(max(self.L.km_emu_num_voxels(self.h), 1), np.int32)
        n = self.L.kocc_emu_evidence(self.h, out.ctypes.data)
        return None if n < 0 else out[:n]

    def add(self, pts, pose=None):
        p = _f64(pts)
        assert self.L.kocc_emu_add_points(self.h, p.ctypes.data, len(p), None if pose is None else _f64(pose).ctypes.data) == 0

    def remove_far(self, origin):
        assert self.L.kocc_emu_remove_far(self.h, _f64(origin).ctypes.data) == 0

    def load(self, voxels):
        keys, counts, pts = np.ascontiguousarray(voxels[0], np.int32), np.ascontiguousarray(voxels[1], np.int32), _f64(voxels[2])
        assert self.L.kocc_emu_load(self.h, keys.ctypes.data, counts.ctypes.data, pts.ctypes.data, len(counts)) == 0

    def clear(self, pts, pose, origin, margin, mm):
        pts, pose, origin = _f64(pts), _f64(pose), _f64(origin)
        st = np.zeros(5, np.int64)
        assert self.L.kocc_emu_clear(self.h, pts.ctypes.data, len(pts), pose.ctypes.data, origin.ctypes.data, margin, mm, self.grid,
                                     st.ctypes.data) == 0
        return dict(zip(STAT_KEYS, st.tolist()))

    def frame(self, pts, n_actual, pose, status, origin=(0.0, 0.0, 0.0), margin=0.0, mm=0):
        pts, pose, origin = _f64(pts), _f64(pose), _f64(origin)
        st = np.zeros(5, np.int64)
        assert self.L.kocc_emu_update_pose_async(self.h, pts.ctypes.data, len(pts), n_actual, pose.ctypes.data, status, origin.ctypes.data,
                                                 margin, mm, self.grid, st.ctypes.data) == 0
        return dict(zip(STAT_KEYS, st.tolist()))

    def consistent(self):
        out = [np.zeros((1 << 20, 4), np.int32) for _ in range(2)]
        n = [self.L.kpm_emu_table(self.h, f, out[f].ctypes.data, len(out[f])) for f in (0, 1)]
        tables = sorted(map(tuple, out[0][:n[0]].tolist())) == sorted(map(tuple, out[1][:n[1]].tolist()))
        return tables and self.L.kpm_emu_spare_mirrors_prior(self.h) == 1 and self.L.kocc_emu_spare_mirrors_prior(self.h) == 1

    def close(self):
        self.L.kpm_emu_thaw(self.h)
        self.L.kocc_emu_set(self.h, 0, 0, 0, 0)
        self.L.km_emu_destroy(self.h)


def _scene(seed):
    """a wall at x ~ 12 m, a 'van' of live voxels in front of it, clutter around; rays from near the origin to the wall"""
    rng = np.random.default_rng(seed)
    wall = np.c_[np.full(1500, 12.2) + rng.uniform(0, 0.2, 1500), rng.uniform(-6, 6, 1500), rng.uniform(-1, 2, 1500)]
    van = np.c_[rng.uniform(5, 7, 800), rng.uniform(-1.5, 1.5, 800), rng.uniform(-0.5, 1.5, 800)]
    clutter = rng.uniform(-10, 10, (600, 3))
    rays = np.c_[np.full(900, 12.3) + rng.uniform(0, 0.05, 900), rng.uniform(-5, 5, 900), rng.uniform(-0.8, 1.8, 900)]
    return [np.round(a * 1024) / 1024 for a in (wall, van, clutter, rays)]


class _Expect:
    """the oracle's state beside the emulated map: export, evidence, P"""

    def __init__(self, m, occ):
        self.m, self.occ = m, occ
        self.vox, self.ev = m.export(), None

    def check(self):
        got = self.m.export()
        assert _bytes(got) == _bytes(self.vox)
        ev = self.m.evidence()
        assert (ev is None) == (self.ev is None)
        if ev is not None:
            assert ev.tobytes() == np.ascontiguousarray(self.ev, np.int32).tobytes()
        assert self.m.consistent()

    def carried(self):
        """after an insert or an eviction: the map's new export, evidence carried by key"""
        after = self.m.export()
        if self.ev is not None:
            self.ev = O.carry(self.vox[0], self.ev, after[0], self.occ[0])
        self.vox = after
        self.check()

    def clear(self, oracle, rays, pose, origin, margin, mm):
        want, wev, wst = O.clear(oracle, self.vox, self.ev, self.m.P(), VS, MD, rays, pose, origin, margin, mm, self.occ)
        st = self.m.clear(rays, pose, origin, margin, mm)
        assert st == wst
        self.vox, self.ev = want, wev
        self.check()
        return st


@pytest.mark.parametrize("grid", [1, 3, 0])
@pytest.mark.parametrize("prior", [False, True])
def test_sequence_matches_the_oracle(oracle, grid, prior):
    L = _lib()
    wall, van, clutter, rays = _scene(1)
    occ = (2, 1, 1, 3)
    m = _Map(L, grid)
    try:
        m.set(occ)
        x = _Expect(m, occ)
        m.add(np.concatenate([wall, clutter]))
        x.ev = np.full(0, 2, np.int32)
        x.carried()
        assert set(x.ev.tolist()) == {2}
        if prior:
            L.kocc_emu_freeze(m.h)
            assert m.P() == len(x.vox[1])
            x.check()
        m.add(van)
        x.carried()
        cleared = 0
        for margin, mm in ((0.5, 2), (0.0, 1), (0.25, 2)):
            cleared += x.clear(oracle, rays, POSE, ORIGIN, margin, mm)["cleared_voxels"]
        assert cleared > 0 and len(set(x.ev.tolist())) > 1  # evidence moved and some voxels left
        m.add(van[::3], POSE)  # the van seen again, through a pose: new voxels start at initial, old ones keep their evidence
        x.carried()
        x.clear(oracle, rays[::2], POSE, ORIGIN, 0.5, 2)
        m.remove_far([40.0, 0.0, 0.0])  # the far side of the clutter is evicted (never the prior)
        x.carried()
        x.clear(oracle, rays, POSE, ORIGIN, 0.5, 1)
        if prior:
            L.kpm_emu_thaw(m.h)
            x.check()
            st = x.clear(oracle, rays, POSE, ORIGIN, 0.5, 1)
            assert st["prior_contradicted"] == 0
        m.set(occ)  # a set call resets every voxel to initial
        x.ev = np.full(len(x.vox[1]), occ[0], np.int32)
        x.check()
        x.clear(oracle, rays, POSE, ORIGIN, 0.25, 2)
        voxels = x.vox
        m.load(voxels)
        x.vox, x.ev = voxels, np.full(len(voxels[1]), occ[0], np.int32)
        x.check()
        x.clear(oracle, rays, POSE, ORIGIN, 0.0, 1)
        m.set(None)  # off: memoryless
        x.ev, x.occ = None, None
        x.check()
        x.clear(oracle, rays, POSE, ORIGIN, 0.0, 1)
    finally:
        m.close()


def test_1_0_1_1_equals_memoryless_clearing(oracle):
    L = _lib()
    wall, van, clutter, rays = _scene(2)
    a, b = _Map(L), _Map(L)
    try:
        a.set((1, 0, 1, 1))
        a.add(np.concatenate([wall, clutter, van]))
        for margin, mm in ((0.5, 2), (0.0, 1), (0.25, 3), (0.0, 1)):
            b.load(a.export())  # the emulated inserts create blocks in a racy order: b takes a's
            sa, sb = a.clear(rays, POSE, ORIGIN, margin, mm), b.clear(rays, POSE, ORIGIN, margin, mm)
            assert sa == sb
            assert _bytes(a.export()) == _bytes(b.export())
            assert set(a.evidence().tolist()) <= {1}
            a.add(van[::5])
    finally:
        a.close()
        b.close()


def _by_key(voxels, evidence):
    """(key, points bytes, evidence) per voxel, sorted by key: the emulated inserts create blocks in a racy order, so two maps fed the
    same points agree voxel by voxel, not block by block"""
    keys, counts, pts = voxels
    starts = np.r_[0, np.cumsum(counts)[:-1]].astype(np.int64)
    order = np.lexsort(np.asarray(keys).T[::-1])
    return [(tuple(keys[v]), pts[starts[v]:starts[v] + counts[v]].tobytes(), int(evidence[v])) for v in order]


@pytest.mark.parametrize("prior", [False, True])
def test_frame_path_equals_option_off_frame_then_the_oracle(oracle, prior):
    L = _lib()
    wall, van, clutter, rays = _scene(4)
    occ = (3, 2, 1, 5)
    frame = np.concatenate([rays, wall[:300]])
    origin = [0.2, 0.0, 0.4]
    a, b = _Map(L), _Map(L)
    try:
        for m in (a, b):
            m.set(occ)
            m.add(np.concatenate([wall, clutter]))
            if prior:
                L.kocc_emu_freeze(m.h)
            m.add(van)
        total = 0
        for k, (dx, n_cut, status) in enumerate(((0.0, 17, 0), (0.3, 0, 0), (0.0, 5, 3), (-0.2, 40, 0), (0.1, 0, 0))):
            pose = POSE.copy()
            pose[4] += dx
            n_actual = len(frame) - n_cut
            before = a.export(), a.evidence()
            st = a.frame(frame, n_actual, pose, status, origin, 0.5, 2)
            b.frame(frame, n_actual, pose, status)
            if status != 0:
                assert st == dict.fromkeys(STAT_KEYS, 0)
                assert _bytes(a.export()) == _bytes(before[0]) and a.evidence().tobytes() == before[1].tobytes()
                assert a.consistent()
                continue
            want, wev, wst = O.clear(oracle, b.export(), b.evidence(), b.P(), VS, MD, frame[:n_actual], pose, origin, 0.5, 2, occ)
            assert st == wst, k
            got = a.export()
            assert _by_key(got, a.evidence()) == _by_key(want, wev), k
            P = a.P()  # the prior and its evidence never move or change
            assert _bytes((got[0][:P], got[1][:P])) == _bytes((before[0][0][:P], before[0][1][:P]))
            assert a.evidence()[:P].tobytes() == before[1][:P].tobytes()
            assert a.consistent()
            # b follows with the standalone call, which the sequence test holds to the oracle
            assert b.clear(frame[:n_actual], pose, origin, 0.5, 2) == wst
            assert _bytes(b.export()) == _bytes(want) and b.evidence().tobytes() == wev.tobytes()
            total += wst["cleared_voxels"] + wst["prior_contradicted"]
        assert total > 0
    finally:
        a.close()
        b.close()
