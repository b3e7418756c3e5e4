"""The map-update gate under the SIMT emulator: k_map_update_gate (kicp_map_update_kernels.cuh) at several launch shapes against the
Python rule on the boundary table, its shadow block carrying the registration's pose and a status that is KICP_OK exactly when the
update is applied; then the frame's map-update sequence (km_emu_update_pose_async, the launches of kicp_map_update_pose_async) driven
by an APPLIED shadow block equals the Update at the registration's pose, and driven by a REJECTED one leaves export_voxels bit-identical."""
import ctypes as C

import numpy as np

import map_update_rule as R
from emu import harness as H


def _lib():
    L = H.build("kmu_emu")
    L.kmu_emu_gate.restype = C.c_int32
    L.kmu_emu_gate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    return L


def _gate(L, policy, status, empty, st, pose, grid=1, threads=1):
    from kinematic_icp_b200 import _capi
    res = _capi.RegResult()
    res.pose[:] = list(pose)
    res.status = status
    s = _capi.CorrStats()
    s.n_points, s.n_inliers, s.fitness, s.inlier_rmse = st
    p = _capi.MapUpdatePolicy(*policy)
    shadow = _capi.RegResult()
    shadow.status = -7
    out = C.c_int32(-1)
    assert L.kmu_emu_gate(C.addressof(res), C.addressof(s), C.addressof(p), 1 if empty else 0, grid, threads, C.addressof(shadow),
                          C.byref(out)) == 0
    return out.value, shadow


def test_gate_kernel_table():
    L = _lib()
    pose = [0.0, 0.0, np.sin(0.1), np.cos(0.1), 1.5, -2.0, 0.25]
    for grid, threads in ((1, 1), (1, 32), (2, 64)):
        for policy, status, empty, st in R.table():
            if policy[0] == R.NEVER:
                continue  # NEVER launches no gate
            o, shadow = _gate(L, policy, status, empty, st, pose, grid, threads)
            assert o == R.rule(*policy, status, empty, st[1], st[2], st[3]), (policy, status, empty, st, o)
            assert list(shadow.pose) == pose
            assert shadow.status == (R.KICP_OK if o == R.APPLIED else R.KICP_WARN_NO_CORRESPONDENCES)


def _sorted(voxels):
    """the voxels by key, each with its points in insertion order (the block order follows the emulated threads' atomics)"""
    keys, counts, pts = voxels
    starts = np.r_[0, np.cumsum(counts)[:-1]]
    order = np.lexsort(keys.T[::-1])
    return [(tuple(keys[v]), pts[starts[v]:starts[v] + counts[v]].tobytes()) for v in order]


def _world(seed, n=3000):
    rng = np.random.default_rng(seed)
    return np.round(np.c_[rng.uniform(-20, 20, n), rng.uniform(-20, 20, n), rng.uniform(-2, 3, n)] * 1024.0) / 1024.0 + 0.0


def test_update_sequence_with_the_shadow_block():
    L = _lib()
    base = _world(1)
    frame = _world(2, 2000)
    pose = np.array([0.0, 0.0, np.sin(0.05), np.cos(0.05), 0.75, -0.5, 0.0])
    gate = (R.GATED, 100, 0.5, 0.25)
    maps = [H.EmuMap(1.0, 30.0, 20) for _ in range(3)]
    try:
        for m in maps:
            m.add_points(base)
        before = maps[2].export_voxels()
        # the reference: the frame's Update at the registration's pose
        maps[0].update_pose_async(frame, len(frame) - 17, pose, 0)
        o, shadow = _gate(L, gate, R.KICP_OK, False, (1000, 900, 0.9, 0.1), pose)
        assert o == R.APPLIED and shadow.status == R.KICP_OK
        maps[1].update_pose_async(frame, len(frame) - 17, np.array(shadow.pose[:]), shadow.status)
        assert _sorted(maps[0].export_voxels()) == _sorted(maps[1].export_voxels())
        assert maps[1].num_points() == maps[0].num_points() != len(before[2])  # the frame did change the map
        o, shadow = _gate(L, gate, R.KICP_OK, False, (1000, 900, 0.9, 0.3), pose)
        assert o == R.REJECTED and shadow.status != R.KICP_OK
        maps[2].update_pose_async(frame, len(frame) - 17, np.array(shadow.pose[:]), shadow.status)
        after = maps[2].export_voxels()
        assert all(x.tobytes() == y.tobytes() for x, y in zip(before, after))
        assert maps[2].num_points() == len(before[2]) and maps[2].num_voxels() == len(before[1])
    finally:
        for m in maps:
            m.close()
