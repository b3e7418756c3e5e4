"""The map kernels with a frozen prior prefix under the SIMT emulator (tests/emu/kpm_emu.cpp: the launch sequences of kicp_map.cu with
prior_blocks = P), against the oracle of tests/prior_map_oracle.py: the synchronous sequence (AddPoints, RemovePointsFarFromLocation,
Update) and the frame path's sequence after every step, a result block that is not KICP_OK leaving the map bit-identical, the spare
arrays holding the mirrored prefix across compactions, and the table restored from the snapshot plus the suffix holding exactly the
entries of a table rebuilt from every block."""
import ctypes as C

import numpy as np

from emu import harness as H
from prior_map_oracle import PriorMap


def _lib():
    L = H.build("kpm_emu")
    H.km_lib()  # the typed km_emu_* entry points (the same source is compiled into both)
    L.km_emu_create.restype = C.c_void_p
    L.km_emu_create.argtypes = [C.c_double, C.c_double, C.c_int32, C.c_uint32]
    L.km_emu_destroy.argtypes = [C.c_void_p]
    for f in (L.km_emu_num_points, L.km_emu_num_voxels):
        f.restype, f.argtypes = C.c_int64, [C.c_void_p]
    L.km_emu_export.restype = C.c_int64
    L.km_emu_export.argtypes = [C.c_void_p] * 4
    L.km_emu_add_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    for f in (L.kpm_emu_freeze, L.kpm_emu_thaw):
        f.argtypes = [C.c_void_p]
    L.kpm_emu_prior_blocks.restype = C.c_uint32
    L.kpm_emu_prior_blocks.argtypes = [C.c_void_p]
    L.kpm_emu_add_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    L.kpm_emu_remove_far.argtypes = [C.c_void_p, C.c_void_p]
    L.kpm_emu_update_pose_async.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32]
    L.kpm_emu_spare_mirrors_prior.argtypes = [C.c_void_p]
    L.kpm_emu_table.restype = C.c_int64
    L.kpm_emu_table.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]
    return L


class _Map:
    def __init__(self, L, vs=1.0, md=30.0, cap=20, blocks_cap=60000):
        self.L = L
        self.h = C.c_void_p(L.km_emu_create(vs, md, cap, blocks_cap))

    def export(self):
        nv, npts = self.L.km_emu_num_voxels(self.h), self.L.km_emu_num_points(self.h)
        keys, counts, pts = np.zeros((nv, 3), np.int32), np.zeros(nv, np.int32), np.zeros((npts, 3))
        assert self.L.km_emu_export(self.h, keys.ctypes.data, counts.ctypes.data, pts.ctypes.data) == nv
        return keys, counts, pts

    def add(self, pts, pose=None):
        pts = np.ascontiguousarray(pts, dtype=np.float64)
        p = None if pose is None else np.ascontiguousarray(pose, dtype=np.float64)
        assert self.L.kpm_emu_add_points(self.h, pts.ctypes.data, len(pts), None if p is None else p.ctypes.data) == 0

    def remove_far(self, origin):
        o = np.ascontiguousarray(origin, dtype=np.float64)
        assert self.L.kpm_emu_remove_far(self.h, o.ctypes.data) == 0

    def update_pose_async(self, pts, n_actual, pose, status=0):
        pts = np.ascontiguousarray(pts, dtype=np.float64)
        p = np.ascontiguousarray(pose, dtype=np.float64)
        assert self.L.kpm_emu_update_pose_async(self.h, pts.ctypes.data, len(pts), n_actual, p.ctypes.data, status) == 0

    def table(self, fresh):
        out = np.zeros((1 << 20, 4), np.int32)
        n = self.L.kpm_emu_table(self.h, 1 if fresh else 0, out.ctypes.data, len(out))
        assert n >= 0
        return sorted(map(tuple, out[:n].tolist()))

    def close(self):
        self.L.kpm_emu_thaw(self.h)
        self.L.km_emu_destroy(self.h)


def _sorted(voxels):
    keys, counts, pts = voxels
    starts = np.r_[0, np.cumsum(counts)[:-1]]
    order = np.lexsort(keys.T[::-1])
    return [(tuple(keys[v]), pts[starts[v]:starts[v] + counts[v]].tobytes()) for v in order]


def _bytes(v):
    return tuple(np.ascontiguousarray(a).tobytes() for a in v)


def _prefix(v, nv):
    keys, counts, pts = v
    return keys[:nv], counts[:nv], pts[:int(counts[:nv].sum())]


def _world(seed, n=3000, half=20.0, dx=0.0):
    rng = np.random.default_rng(seed)
    return np.round(np.c_[rng.uniform(-half, half, n) + dx, rng.uniform(-half, half, n), rng.uniform(-2, 3, n)] * 1024.0) / 1024.0 + 0.0


def _check(m, om, prior, step):
    got = m.export()
    assert _sorted(got) == _sorted(om.export_voxels()), step
    P = len(prior[1])
    assert _bytes(_prefix(got, P)) == _bytes(prior), step
    assert m.L.kpm_emu_spare_mirrors_prior(m.h) == 1, step
    assert m.table(False) == m.table(True), step


def test_synchronous_sequence(oracle):
    ko = oracle
    L = _lib()
    m = _Map(L)
    try:
        m.add(np.concatenate([_world(1, 3000, 15.0), _world(2, 800, 3.0, dx=90.0)]))  # a far patch: beyond max_distance below
        L.kpm_emu_freeze(m.h)
        prior = m.export()
        om = PriorMap(ko, prior, 1.0, 30.0, 20)
        pose = np.array([0.0, 0.0, np.sin(0.2), np.cos(0.2), 5.0, -3.0, 0.0])
        m.add(_world(3, 2000, 30.0))
        om.add_points(_world(3, 2000, 30.0))
        _check(m, om, prior, "add")
        m.remove_far([-20.0, 0.0, 0.0])
        om.remove_far([-20.0, 0.0, 0.0])
        _check(m, om, prior, "remove_far")
        m.add(_world(4, 2000, 30.0), pose)
        m.remove_far(pose[4:])
        om.update_pose(_world(4, 2000, 30.0), pose)
        _check(m, om, prior, "update_pose")
        assert om.live.num_voxels() > 0
    finally:
        m.close()


def test_frame_path_sequence_and_untouched_on_a_failed_result(oracle):
    ko = oracle
    L = _lib()
    m = _Map(L)
    try:
        m.add(np.concatenate([_world(5, 3000, 15.0), _world(6, 800, 3.0, dx=90.0)]))
        L.kpm_emu_freeze(m.h)
        prior = m.export()
        om = PriorMap(ko, prior, 1.0, 30.0, 20)
        for k, (tx, yaw) in enumerate(((0.0, 0.0), (8.0, 0.3), (25.0, -0.4))):
            frame = _world(10 + k, 2500, 25.0)
            pose = np.array([0.0, 0.0, np.sin(yaw / 2), np.cos(yaw / 2), tx, 1.0, 0.0])
            m.update_pose_async(frame, len(frame) - 13, pose, 0)
            om.update_pose(frame[:len(frame) - 13], pose)
            _check(m, om, prior, k)
        before = m.export()
        frame = _world(20, 2000, 25.0)
        m.update_pose_async(frame, len(frame), np.array([0.0, 0.0, 0.0, 1.0, -40.0, 0.0, 0.0]), 3)  # NaN pose / gated off
        assert _bytes(m.export()) == _bytes(before)
        assert m.table(False) == m.table(True)
    finally:
        m.close()


def test_thaw_resumes_the_plain_sequence(oracle):
    """after thaw the same emulated map runs the plain launch sequences (P = 0): the far prior voxels die at the next eviction"""
    ko = oracle
    L = _lib()
    m = _Map(L)
    try:
        m.add(np.concatenate([_world(7, 2000, 10.0), _world(8, 500, 3.0, dx=90.0)]))
        L.kpm_emu_freeze(m.h)
        m.remove_far([0.0, 0.0, 0.0])
        assert any(k[0] >= 80 for k in m.export()[0].tolist())
        L.kpm_emu_thaw(m.h)
        assert L.kpm_emu_prior_blocks(m.h) == 0
        m.remove_far([0.0, 0.0, 0.0])
        assert not any(k[0] >= 80 for k in m.export()[0].tolist())
        assert m.table(False) == m.table(True)
    finally:
        m.close()
