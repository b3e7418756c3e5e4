"""Occupancy evidence without a GPU: the oracle of tests/occupancy_oracle.py on hand-built, binary-exact cases (how many free calls a
voxel survives, the clamp at max_evidence, hit_gain 0, a prior's evidence, ray order, and {1, 0, 1, 1} against the memoryless rule of
free_space_oracle.py); the header, the ctypes mirror and the Python defaults; every argument check of the new calls that fails before
any device work, with its text; and kicp_replay's refusal of --occupancy without --free-space or with a malformed value."""
import os
import re
import subprocess

import numpy as np
import pytest

import free_space_oracle as F
import occupancy_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
I7 = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
ORIGIN = [0.5, 0.5, 0.5]
# voxel (2, 0, 0) in front of a wall at x = 6; THROUGH passes it three times (each ray ends in its own wall voxel), HIT ends in it
WALL = [[2, 0, 0], [6, 0, 0], [6, 1, 0], [6, -1, 0]]
THROUGH = [[6.5, 0.5, 0.5], [6.5, 1.2, 0.5], [6.5, -0.2, 0.5]]
HIT = [[2.5, 0.5, 0.5]]


def _build():
    import __graft_entry__ as g
    g.build()


def _map(keys, v=1.0):
    """an export with one point at the centre of every voxel"""
    keys = np.asarray(keys, np.int32).reshape(-1, 3)
    return keys, np.ones(len(keys), np.int32), (keys + 0.5) * v


def _keys(vox):
    return [tuple(k) for k in vox[0].tolist()]


def _call(ko, vox, ev, rays, occ, P=0, mm=2, v=1.0, margin=0.0, pose=I7, origin=ORIGIN):
    return O.clear(ko, vox, ev, P, v, 100.0, rays, pose, origin, margin, mm, occ)


@pytest.mark.parametrize("occ,k", [((1, 1, 1, 8), 0), ((1, 1, 1, 8), 3), ((2, 3, 2, 16), 2), ((3, 2, 4, 9), 4), ((5, 0, 2, 5), 7)])
def test_a_voxel_survives_ceil_e_over_loss_minus_one_free_calls(oracle, occ, k):
    initial, gain, loss, top = occ
    vox = _map(WALL)
    ev = np.full(len(WALL), initial, np.int32)
    for _ in range(k):  # k calls whose ray ends in the voxel
        vox, ev, st = _call(oracle, vox, ev, HIT, occ)
        assert st["cleared_voxels"] == 0
    e = min(initial + k * gain, top)
    assert int(ev[0]) == e
    survive = O.calls_to_clear(e, loss)
    assert survive == -(-e // loss) - 1
    for c in range(survive):
        vox, ev, st = _call(oracle, vox, ev, THROUGH, occ)
        assert (2, 0, 0) in _keys(vox) and st["cleared_voxels"] == 0, c
        assert int(ev[0]) == e - (c + 1) * loss > 0
    vox, ev, st = _call(oracle, vox, ev, THROUGH, occ)
    assert (2, 0, 0) not in _keys(vox)
    assert st["cleared_voxels"] == 1 and st["cleared_points"] == 1
    assert len(ev) == 3


def test_clamped_at_max_evidence(oracle):
    occ = (2, 5, 1, 4)
    vox = _map(WALL)
    ev = np.full(len(WALL), 2, np.int32)
    vox, ev, _ = _call(oracle, vox, ev, HIT, occ)
    assert ev.tolist() == [4, 2, 2, 2]
    vox, ev, _ = _call(oracle, vox, ev, HIT * 3, occ)  # three hits in one call: one update
    assert ev.tolist() == [4, 2, 2, 2]
    # the wall voxels are hit by THROUGH: clamped as well; (2, 0, 0) loses one per call
    vox, ev, _ = _call(oracle, vox, ev, THROUGH, occ)
    assert ev.tolist() == [3, 4, 4, 4]


def test_hit_gain_zero_only_keeps_the_evidence(oracle):
    occ = (2, 0, 1, 8)
    vox = _map(WALL)
    ev = np.full(len(WALL), 2, np.int32)
    for _ in range(5):
        vox, ev, _ = _call(oracle, vox, ev, HIT, occ)
    assert ev.tolist() == [2, 2, 2, 2]
    vox, ev, st = _call(oracle, vox, ev, THROUGH, occ)
    assert st["cleared_voxels"] == 0 and int(ev[0]) == 1
    vox, ev, st = _call(oracle, vox, ev, THROUGH, occ)
    assert st["cleared_voxels"] == 1 and _keys(vox) == [(6, 0, 0), (6, 1, 0), (6, -1, 0)]


def test_prior_evidence_is_untouched_while_prior_contradicted_is_counted(oracle):
    occ = (1, 1, 1, 4)
    vox = _map([[2, 0, 0], [3, 0, 0], [6, 0, 0], [6, 1, 0], [6, -1, 0]])
    ev = np.array([1, 1, 1, 1, 1], np.int32)
    for _ in range(4):  # (2, 0, 0) is prior (P = 1); (3, 0, 0) is live and crossed by the same rays
        vox, ev, st = _call(oracle, vox, ev, THROUGH, occ, P=1)
        assert st["prior_contradicted"] == 1
    assert _keys(vox)[0] == (2, 0, 0) and int(ev[0]) == 1
    assert (3, 0, 0) not in _keys(vox)
    vox, ev, st = _call(oracle, vox, ev, HIT, occ, P=1)  # a hit on a prior voxel does not raise it either
    assert int(ev[0]) == 1 and st["prior_contradicted"] == 0


def test_result_does_not_depend_on_the_order_of_the_rays(oracle):
    rng = np.random.default_rng(5)
    keys = np.unique(rng.integers(-8, 8, (400, 3)), axis=0)
    vox = _map(keys, 0.5)
    ev = rng.integers(1, 4, len(keys)).astype(np.int32)
    pts = rng.uniform(-4, 4, (500, 3))
    pose = np.array([0.0, 0.0, np.sin(0.15), np.cos(0.15), 0.3, -0.2, 0.1])
    occ = (2, 1, 1, 3)
    a = O.clear(oracle, vox, ev, 40, 0.5, 100.0, pts, pose, [0.1, 0.0, 0.2], 0.25, 2, occ)
    b = O.clear(oracle, vox, ev, 40, 0.5, 100.0, pts[rng.permutation(len(pts))], pose, [0.1, 0.0, 0.2], 0.25, 2, occ)
    assert a[2] == b[2] and a[2]["cleared_voxels"] > 0
    assert np.array_equal(a[1], b[1])
    assert all(np.array_equal(x, y) for x, y in zip(a[0], b[0]))


def _scenes():
    """the scenes of test_free_space_cpu.py: (voxels, P, voxel size, points, pose, origin, margin, min_misses)"""
    rng = np.random.default_rng(5)
    keys = np.unique(rng.integers(-8, 8, (400, 3)), axis=0)
    pose = np.array([0.0, 0.0, np.sin(0.15), np.cos(0.15), 0.3, -0.2, 0.1])
    pts = [[np.nan, 0.5, 0.5], [np.inf, 0.5, 0.5], [1e300, 0.5, 0.5], [-3e9, 0.5, 0.5], [3.5, 0.5, 0.5]]
    return [(_map([[0, 0, 0], [1, 0, 0]]), 0, 1.0, [[0.5, 0.5, 0.5]], I7, ORIGIN, 0.0, 1),
            (_map([[1, 0, 0], [2, 0, 0]]), 0, 1.0, pts, I7, ORIGIN, 0.0, 1),
            (_map(WALL), 0, 1.0, THROUGH, I7, ORIGIN, 0.0, 3),
            (_map(WALL), 0, 1.0, THROUGH, I7, ORIGIN, 0.0, 4),
            (_map([[2, 0, 0], [3, 0, 0], [6, 0, 0]]), 0, 1.0, [[6.5, 0.5, 0.5], [6.5, 0.5, 0.5], [3.5, 0.5, 0.5]], I7, ORIGIN, 0.0, 2),
            (_map([[2, 0, 0], [3, 0, 0], [6, 0, 0]]), 1, 1.0, [[6.5, 0.5, 0.5], [6.5, 0.5, 0.5], [3.5, 0.5, 0.5]], I7, ORIGIN, 0.0, 2),
            (_map(keys, 0.5), 40, 0.5, rng.uniform(-4, 4, (500, 3)), pose, [0.1, 0.0, 0.2], 0.25, 2)]


def test_1_0_1_1_is_the_memoryless_rule(oracle):
    for vox, P, v, pts, pose, origin, margin, mm in _scenes():
        ev = np.ones(len(vox[1]), np.int32)
        want, wst = F.clear_free_space(oracle, vox, P, v, 100.0, pts, pose, origin, margin, mm)
        got, gev, gst = O.clear(oracle, vox, ev, P, v, 100.0, pts, pose, origin, margin, mm, (1, 0, 1, 1))
        assert gst == wst
        assert all(np.array_equal(a, b) for a, b in zip(got, want))
        assert gev.tolist() == [1] * len(got[1])
        off, oev, ost = O.clear(oracle, vox, None, P, v, 100.0, pts, pose, origin, margin, mm, None)
        assert ost == wst and oev is None and all(np.array_equal(a, b) for a, b in zip(off, want))


def test_carry_keeps_evidence_by_key_and_new_voxels_start_at_initial():
    before = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0]])
    after = np.array([[0, 0, 0], [2, 0, 0], [5, 5, 5]])
    assert O.carry(before, [3, 1, 7], after, 2).tolist() == [3, 7, 2]


def test_header_mirror_and_defaults():
    from kinematic_icp_b200 import _capi
    import kinematic_icp_b200 as K
    hdr = open(os.path.join(ROOT, "include", "kicp.h")).read()
    body = re.search(r"typedef struct kicp_occupancy_params \{(.*?)\} kicp_occupancy_params;", hdr, re.S).group(1)
    fields = re.findall(r"int32_t (\w+);", body)
    assert fields == [f for f, _ in _capi.OccupancyParams._fields_] == ["initial", "hit_gain", "miss_loss", "max_evidence"]
    for name in ("kicp_map_set_occupancy", "kicp_map_export_occupancy"):
        assert re.search(r"\bint %s\(" % name, hdr), name
        assert name in {s[0] for s in _capi.SYMBOLS}, name
    d = (K.OCCUPANCY_INITIAL, K.OCCUPANCY_HIT_GAIN, K.OCCUPANCY_MISS_LOSS, K.OCCUPANCY_MAX_EVIDENCE)
    assert 1 <= d[0] <= d[3] <= 1 << 24 and 0 <= d[1] <= 1 << 24 and 1 <= d[2] <= 1 << 24


def test_validation():
    """every check before the map is reachable with a null map (no device); the map last"""
    import ctypes as C
    _build()
    from kinematic_icp_b200 import _capi
    lib = _capi.lib()

    def err(rc, fn, text):
        assert rc == _capi.KICP_ERR_INVALID, rc
        assert lib.kicp_last_error().decode() == "%s: %s" % (fn, text)

    fn = "kicp_map_set_occupancy"
    for p, text in (((1, 0, 1, 0), "params->max_evidence: outside [1, 2^24]"),
                    ((1, 0, 1, (1 << 24) + 1), "params->max_evidence: outside [1, 2^24]"),
                    ((0, 0, 1, 4), "params->initial: outside [1, max_evidence]"),
                    ((5, 0, 1, 4), "params->initial: outside [1, max_evidence]"),
                    ((1, -1, 1, 4), "params->hit_gain: outside [0, 2^24]"),
                    ((1, (1 << 24) + 1, 1, 4), "params->hit_gain: outside [0, 2^24]"),
                    ((1, 0, 0, 4), "params->miss_loss: outside [1, 2^24]"),
                    ((1, 0, (1 << 24) + 1, 4), "params->miss_loss: outside [1, 2^24]")):
        err(lib.kicp_map_set_occupancy(None, C.byref(_capi.OccupancyParams(*p))), fn, text)
    err(lib.kicp_map_set_occupancy(None, C.byref(_capi.OccupancyParams(1 << 24, 1 << 24, 1 << 24, 1 << 24))), fn, "null map")
    err(lib.kicp_map_set_occupancy(None, None), fn, "null map")
    n = C.c_int64()
    err(lib.kicp_map_export_occupancy(None, None, 0, None), "kicp_map_export_occupancy", "n: null pointer")
    err(lib.kicp_map_export_occupancy(None, None, 0, C.byref(n)), "kicp_map_export_occupancy", "null map")


def test_replay_refuses_occupancy_without_free_space_or_malformed(tmp_path):
    _build()
    exe = os.path.join(ROOT, "kinematic-icp_b200", "bin", "kicp_replay")
    base = [exe, str(tmp_path / "none.kseq"), str(tmp_path / "x.tum")]
    out = subprocess.run(base + ["--occupancy", "2,1,1,4"], capture_output=True, text=True, timeout=60)
    assert out.returncode == 2 and "--occupancy" in out.stderr and "--free-space" in out.stderr
    for bad in ("2,1,1", "2,1,1,4,5", "a,1,1,4", "2,,1,4", "2,1,1,4x", ""):
        out = subprocess.run(base + ["--free-space", "2", "--occupancy", bad], capture_output=True, text=True, timeout=60)
        assert out.returncode == 2 and "--occupancy takes I,G,L,M" in out.stderr, bad
