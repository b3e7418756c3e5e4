"""The frame path's map-update policy without a GPU: kicp_map_update_policy as gcc lays it out against its ctypes mirror and the
constants against the header; every argument check of kicp_ctx_set_map_update and kicp_frame_map_update with its text (the context is
checked last, so each is reachable without a device); the rule of kicp_map_update.h, compiled for the host, against the Python
restatement at its exact boundaries; and kicp_replay's map file (kicp/map_file.hpp) against a numpy reader, corrupt files included."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

import map_update_rule as R
from emu import harness as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build():
    import __graft_entry__ as g
    g.build()


def test_struct_layout_and_constants(tmp_path):
    from kinematic_icp_b200 import _capi
    ct = _capi.MapUpdatePolicy
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "kicp.h"', 'int main(void) {',
             'printf("sizeof %zu\\n", sizeof(kicp_map_update_policy));']
    lines += ['printf("%s %%zu\\n", offsetof(kicp_map_update_policy, %s));' % (f, f) for f, _ in ct._fields_]
    lines += ['return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["sizeof"]) == C.sizeof(ct) == 32
    for f, _ in ct._fields_:
        assert int(out[f]) == getattr(ct, f).offset, f
    hdr = open(os.path.join(ROOT, "include", "kicp.h")).read()
    defs = dict((k, int(v)) for k, v in re.findall(r"#define (KICP_(?:MAP|FRAME)_UPDATE_[A-Z_]+) (\d+)", hdr))
    assert len(defs) == 8
    for k, v in defs.items():
        assert getattr(_capi, k) == v == getattr(R, k.split("_UPDATE_")[1]), k


BAD = [
    (dict(mode=-1), "policy->mode: not in 0..2"),
    (dict(mode=3), "policy->mode: not in 0..2"),
    (dict(min_inliers=-1), "policy->min_inliers: negative"),
    (dict(min_fitness=math.nan), "policy->min_fitness: not in [0, 1]"),
    (dict(min_fitness=-1e-300), "policy->min_fitness: not in [0, 1]"),
    (dict(min_fitness=math.nextafter(1.0, 2.0)), "policy->min_fitness: not in [0, 1]"),
    (dict(max_inlier_rmse=math.nan), "policy->max_inlier_rmse: not > 0"),
    (dict(max_inlier_rmse=0.0), "policy->max_inlier_rmse: not > 0"),
    (dict(max_inlier_rmse=-math.inf), "policy->max_inlier_rmse: not > 0"),
]


def test_validation():
    _build()
    from kinematic_icp_b200 import _capi
    lib = _capi.lib()

    def err(rc, fn, text):
        assert rc == _capi.KICP_ERR_INVALID, rc
        assert lib.kicp_last_error().decode() == "%s: %s" % (fn, text)

    fn = "kicp_ctx_set_map_update"
    err(lib.kicp_ctx_set_map_update(None, None), fn, "policy: null pointer")
    good = dict(mode=2, min_inliers=0, min_fitness=0.0, max_inlier_rmse=math.inf)
    for kw, text in BAD:
        p = _capi.MapUpdatePolicy(**dict(good, **kw))
        err(lib.kicp_ctx_set_map_update(None, C.byref(p)), fn, text)
    for kw in (good, dict(good, mode=0), dict(good, mode=1, min_fitness=1.0, max_inlier_rmse=5e-324), dict(good, min_inliers=1 << 62)):
        p = _capi.MapUpdatePolicy(**kw)
        err(lib.kicp_ctx_set_map_update(None, C.byref(p)), fn, "null context")  # every field passed
    err(lib.kicp_frame_map_update(None, None), "kicp_frame_map_update", "outcome: null pointer")
    o = C.c_int32()
    err(lib.kicp_frame_map_update(None, C.byref(o)), "kicp_frame_map_update", "null context")


def _rule_lib():
    L = H.build("kmu_emu")
    L.kmu_rule.restype = C.c_int32
    L.kmu_rule.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
    return L


def _c_args(policy, st):
    from kinematic_icp_b200 import _capi
    p = _capi.MapUpdatePolicy(*policy)
    s = _capi.CorrStats()
    s.n_points, s.n_inliers, s.fitness, s.inlier_rmse = st
    return p, s


def test_rule_table():
    """kicp_map_update.h compiled for the host == the Python rule on every row of the boundary table"""
    L = _rule_lib()
    seen = set()
    for policy, status, empty, st in R.table():
        p, s = _c_args(policy, st)
        got = L.kmu_rule(C.addressof(p), status, 1 if empty else 0, C.addressof(s))
        want = R.rule(*policy, status, empty, st[1], st[2], st[3])
        assert got == want, (policy, status, empty, st, got, want)
        seen.add(got)
    assert seen == {R.APPLIED, R.NO_CORRESPONDENCES, R.REJECTED, R.SKIPPED}
    # the exact boundaries: equality passes, one inlier or one ulp beyond fails
    gate = (R.GATED, 100, 0.5, 0.25)
    assert R.rule(*gate, 0, False, 100, 0.5, 0.25) == R.APPLIED
    assert R.rule(*gate, 0, False, 99, 0.5, 0.25) == R.REJECTED
    assert R.rule(*gate, 0, False, 100, math.nextafter(0.5, 0), 0.25) == R.REJECTED
    assert R.rule(*gate, 0, False, 100, 0.5, math.nextafter(0.25, 1)) == R.REJECTED
    assert R.rule(*gate, 0, True, 0, 0.0, 0.0) == R.APPLIED  # the empty-map clause


# ------------------------------------------------------------------------------------------------ the map file of kicp_replay
def _hooks():
    _build()
    L = C.CDLL(os.path.join(ROOT, "tests", "hooks", "_build", "libkicp_map_update_hooks.so"))
    L.kmu_map_write.argtypes = [C.c_char_p, C.c_double, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_char_p,
                                C.c_int64]
    L.kmu_map_write.restype = C.c_int32
    L.kmu_map_read.argtypes = [C.c_char_p, C.c_char_p, C.c_int64]
    L.kmu_map_read.restype = C.c_void_p
    L.kmu_map_info.argtypes = [C.c_void_p] + [C.c_void_p] * 4
    L.kmu_map_copy.argtypes = [C.c_void_p] * 4
    L.kmu_map_free.argtypes = [C.c_void_p]
    return L


def write_map(L, path, vs, cap, keys, counts, pts):
    keys, counts, pts = (np.ascontiguousarray(a, dt) for a, dt in ((keys, np.int32), (counts, np.int32), (pts, np.float64)))
    err = C.create_string_buffer(256)
    rc = L.kmu_map_write(str(path).encode(), vs, cap, keys.ctypes.data, counts.ctypes.data, pts.ctypes.data, len(counts), len(pts), err, 256)
    assert rc == 0, err.value


def read_map(L, path):
    """(voxel_size, cap, keys, counts, points) through kicp::read_map_file, or the error text"""
    err = C.create_string_buffer(512)
    h = L.kmu_map_read(str(path).encode(), err, 512)
    if not h:
        return err.value.decode()
    vs, cap, nv, np_ = C.c_double(), C.c_uint32(), C.c_int64(), C.c_int64()
    L.kmu_map_info(h, C.byref(vs), C.byref(cap), C.byref(nv), C.byref(np_))
    keys, counts, pts = np.zeros((nv.value, 3), np.int32), np.zeros(nv.value, np.int32), np.zeros((np_.value, 3))
    L.kmu_map_copy(h, keys.ctypes.data, counts.ctypes.data, pts.ctypes.data)
    L.kmu_map_free(h)
    return vs.value, cap.value, keys, counts, pts


def numpy_read(path):
    """the file format as the header of kicp/map_file.hpp documents it"""
    b = open(path, "rb").read()
    assert b[:8] == b"KICPMAP1"
    vs, = np.frombuffer(b, "<f8", 1, 8)
    cap, zero = np.frombuffer(b, "<u4", 2, 16)
    V, P = np.frombuffer(b, "<i8", 2, 24)
    o = 40
    keys = np.frombuffer(b, "<i4", 3 * V, o).reshape(V, 3)
    counts = np.frombuffer(b, "<i4", V, o + 12 * V)
    pts = np.frombuffer(b, "<f8", 3 * P, o + 16 * V).reshape(P, 3)
    assert zero == 0 and len(b) == o + 16 * V + 24 * P
    return float(vs), int(cap), keys, counts, pts


def _voxels(seed=3, nv=50, cap=20):
    rng = np.random.default_rng(seed)
    keys = rng.integers(-1000, 1000, (nv, 3)).astype(np.int32)
    counts = rng.integers(1, cap + 1, nv).astype(np.int32)
    pts = rng.normal(size=(int(counts.sum()), 3)) * 30.0
    return keys, counts, pts


def test_map_file_round_trip(tmp_path):
    L = _hooks()
    keys, counts, pts = _voxels()
    for k, c, p in ((keys, counts, pts), (keys[:0], counts[:0], pts[:0])):
        path = tmp_path / ("m%d.kmap" % len(c))
        write_map(L, path, 0.75, 20, k, c, p)
        vs, cap, k2, c2, p2 = numpy_read(path)
        assert (vs, cap) == (0.75, 20) and np.array_equal(k2, k) and np.array_equal(c2, c) and p2.tobytes() == p.tobytes()
        vs, cap, k3, c3, p3 = read_map(L, path)
        assert (vs, cap) == (0.75, 20) and np.array_equal(k3, k) and np.array_equal(c3, c) and p3.tobytes() == p.tobytes()


def test_map_file_corrupt(tmp_path):
    """each broken invariant is refused with its reason"""
    L = _hooks()
    keys, counts, pts = _voxels(nv=5, cap=4)
    path = tmp_path / "good.kmap"
    write_map(L, path, 1.0, 4, keys, counts, pts)
    good = bytearray(open(path, "rb").read())
    V, P = len(counts), len(pts)

    def variant(name, b):
        p = tmp_path / name
        p.write_bytes(bytes(b))
        return read_map(L, p)

    def patched(off, fmt, value):
        b = good.copy()
        b[off:off + np.dtype(fmt).itemsize] = np.array([value], fmt).tobytes()
        return b

    assert isinstance(variant("same", good), tuple)
    cases = [
        ("magic", b"KICPMAP2" + good[8:], "not a KICPMAP1 file"),
        ("short", good[:30], "shorter than the header"),
        ("truncated", good[:-1], "length does not match V and P"),
        ("longer", good + b"\0", "length does not match V and P"),
        ("v", patched(24, "<i8", V + 1), "length does not match V and P"),
        ("p", patched(32, "<i8", P - 1), "length does not match V and P"),
        ("negative", patched(24, "<i8", -1), "voxel or point count out of range"),
        ("reserved", patched(20, "<u4", 1), "reserved word not 0"),
        ("voxel_size", patched(8, "<f8", 0.0), "voxel_size not > 0"),
        ("count0", patched(40 + 12 * V, "<i4", 0), "a voxel count outside [1, max_points_per_voxel]"),
        ("count_cap", patched(40 + 12 * V, "<i4", 5), "a voxel count outside [1, max_points_per_voxel]"),
    ]
    # a count moved from one voxel to another keeps the sum; one taken away breaks it
    b = good.copy()
    c0 = int(counts[0])
    b[40 + 12 * V:40 + 12 * V + 4] = np.array([c0 - 1 if c0 > 1 else c0 + 1], "<i4").tobytes()
    cases.append(("sum", b, "the voxel counts do not sum to P"))
    for name, data, why in cases:
        got = variant(name, data)
        assert isinstance(got, str) and got.endswith(": " + why), (name, got)
    assert read_map(L, tmp_path / "missing.kmap").startswith("cannot read")
