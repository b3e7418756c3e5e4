"""The pose search without a GPU: the host logic the library and the emulator share (kicp_pose_search.h, through tests/emu/kps_emu.cpp):
level-0 geometry, children and their dedupe, the ranking key and hypothesis poses bit for bit against the Python restatement
(tests/pose_search_oracle.py); kicp_pose_search_params / kicp_pose_hypothesis as gcc lays them out against their ctypes mirrors; and
every argument check of kicp_map_pose_search* with its text (the map is checked last, so each is reachable without a device)."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import pose_search_oracle as PO
from emu import harness as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _hooks():
    L = H.build("kps_emu")
    L.kps_plan.argtypes = [C.POINTER(PO.Params), C.c_int32, C.POINTER(C.c_int64), C.c_void_p, C.POINTER(C.c_int32), C.c_char_p, C.c_int32]
    L.kps_pose.argtypes = [C.POINTER(PO.Params), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.kps_key_less.argtypes = [C.POINTER(PO.Entry), C.POINTER(PO.Entry)]
    L.kps_children.argtypes = [C.POINTER(PO.Params), C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32]
    L.kps_children.restype = C.c_int32
    return L


def _plan(L, p, cap):
    n0, k, scale, err = C.c_int64(), np.zeros(3, np.int32), C.c_int32(), C.create_string_buffer(128)
    rc = L.kps_plan(C.byref(p), cap, C.byref(n0), k.ctypes.data, C.byref(scale), err, 128)
    return rc, n0.value, tuple(k), scale.value, err.value.decode()


def test_level0_geometry():
    L = _hooks()
    for he, st, lv in [((4.0, 4.0, math.pi), (0.5, 0.5, 0.1), 4), ((1.0, 1.0, 0.2), (0.1, 0.1, 0.02), 3), ((0.0, 0.0, 0.0), (1, 1, 1), 1),
                       ((0.29, 0.3, 0.05), (0.1, 0.1, 0.025), 8)]:
        rc, n0, k, scale, err = _plan(L, PO.params(he, st, 0.5, lv, 8), 8)
        kw, sw, _ = PO.plan(he, st, lv)
        assert rc == 0 and err == "" and list(k) == kw and scale == sw
        assert n0 == (2 * kw[0] + 1) * (2 * kw[1] + 1) * (2 * kw[2] + 1)


def test_pose_bits():
    """prior * Delta composed on the host == the Python restatement with math.sin / math.cos, bit for bit"""
    L = _hooks()
    rng = np.random.default_rng(5)
    for _ in range(40):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        prior = np.r_[q, rng.uniform(-500, 500, 3)]
        st = rng.uniform(0.01, 1.0, 3)
        lv = int(rng.integers(1, 9))
        p = PO.params((1.0, 1.0, 1.0), st, 0.5, lv, 4)
        _, _, u = PO.plan((1.0, 1.0, 1.0), st, lv)
        for Lt in [(0, 0, 0), tuple(int(v) for v in rng.integers(-300, 300, 3)), (7, -3, 2 ** (lv - 1) * 31)]:
            got, off = np.zeros(7), np.zeros(3)
            Ls = np.array(Lt, np.int32)
            prior = np.ascontiguousarray(prior)
            L.kps_pose(C.byref(p), prior.ctypes.data, Ls.ctypes.data, got.ctypes.data, off.ctypes.data)
            want, woff = PO.pose(prior, u, Lt)
            assert np.array_equal(got, want) and list(off) == woff, (Lt, got, want)


def test_key():
    L = _hooks()
    E = lambda Lt, c, s, valid=1: PO.Entry((C.c_int32 * 3)(*Lt), valid, c, s)  # noqa: E731
    items = [E((0, 0, 0), 5, 1.0), E((1, 0, 0), 6, 2.0), E((1, 0, 0), 5, 0.5), E((0, 0, -1), 5, 1.0), E((0, 0, 1), 5, 1.0),
             E((1, 1, 0), 5, 1.0), E((-1, 0, 0), 5, 1.0), E((0, 1, 0), 5, 1.0), E((0, -1, 0), 5, 1.0), E((2, 0, 0), 9, 0.1, valid=0),
             E((2 ** 31 - 1, 2 ** 31 - 1, -2 ** 31), 5, 1.0)]
    ref = sorted(range(len(items)), key=lambda i: (not items[i].valid, PO.key(tuple(items[i].L), items[i].n_inl, items[i].sum_sq)))
    for a in range(len(items)):
        for b in range(len(items)):
            assert L.kps_key_less(C.byref(items[a]), C.byref(items[b])) == (ref.index(a) < ref.index(b)), (a, b)


def test_children_and_dedupe():
    """the 26 neighbours at the level's step, without level 0's box points, the points already refined, and repeats"""
    L = _hooks()
    he, st, lv = (0.2, 0.2, 0.1), (0.1, 0.1, 0.1), 3  # scale 4: level 0 = multiples of 4 in [-8, 8] x [-8, 8] x [-4, 4]
    p = PO.params(he, st, 0.5, lv, 4)
    kept = np.array([[0, 0, 0], [4, 0, 0]], np.int32)
    refined = np.array([[2, 2, 2]], np.int32)
    out = np.zeros((200, 3), np.int32)
    n = L.kps_children(C.byref(p), 1, kept.ctypes.data, 2, refined.ctypes.data, 1, out.ctypes.data, 200)
    want = []
    for c in kept:
        for dp in (-1, 0, 1):
            for dx in (-1, 0, 1):
                for dy in (-1, 0, 1):
                    Lt = (int(c[0]) + 2 * dx, int(c[1]) + 2 * dy, int(c[2]) + 2 * dp)
                    in0 = all(v % 4 == 0 for v in Lt) and abs(Lt[0]) <= 8 and abs(Lt[1]) <= 8 and abs(Lt[2]) <= 4
                    if (dp or dx or dy) and not in0 and Lt != (2, 2, 2) and Lt not in want:
                        want.append(Lt)
    assert [tuple(r) for r in out[:n]] == want and n == len(want) < 51  # shared neighbours of the two kept points only once


def test_struct_layouts(tmp_path):
    """sizeof / offsetof of kicp_pose_search_params and kicp_pose_hypothesis (plain C) == the package's ctypes mirrors == the tests'"""
    from kinematic_icp_b200 import _capi
    pairs = {"kicp_pose_search_params": (_capi.PoseSearchParams, PO.Params), "kicp_pose_hypothesis": (_capi.PoseHypothesis, PO.Hypothesis)}
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "kicp.h"', 'int main(void) {']
    for cname, (ct, _) in pairs.items():
        lines.append('printf("%s.sizeof %%zu\\n", sizeof(%s));' % (cname, cname))
        for fname, _ in ct._fields_:
            lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, fname, cname, fname))
    lines += ['return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    for cname, (ct, tt) in pairs.items():
        assert int(out[cname + ".sizeof"]) == C.sizeof(ct) == C.sizeof(tt)
        for (fname, _), (tname, _) in zip(ct._fields_, tt._fields_):
            assert fname == tname
            assert int(out["%s.%s" % (cname, fname)]) == getattr(ct, fname).offset == getattr(tt, fname).offset


GOOD = dict(half_extent=(1.0, 1.0, 0.2), step=(0.1, 0.1, 0.02), tau=0.5, levels=3, keep=8)
BAD = [
    (dict(half_extent=(float("nan"), 1.0, 0.2)), "params->half_extent: not finite"),
    (dict(step=(0.1, float("inf"), 0.02)), "params->step: not finite"),
    (dict(tau=float("nan")), "params->tau: not finite"),
    (dict(half_extent=(1.0, -1.0, 0.2)), "params->half_extent: negative"),
    (dict(half_extent=(1.0, 1.0, 3.2)), "params->half_extent[2]: yaw above pi"),
    (dict(step=(0.1, 0.0, 0.02)), "params->step: not > 0"),
    (dict(tau=0.0), "params->tau: not > 0"),
    (dict(levels=0), "params->levels: not in 1..8"),
    (dict(levels=9), "params->levels: not in 1..8"),
    (dict(keep=0), "params->keep: not in 1..64"),
    (dict(keep=65), "params->keep: not in 1..64"),
    (dict(half_extent=(100.0, 100.0, 0.2), step=(0.01, 0.01, 0.02)), "params: more than 4194304 level-0 hypotheses"),
    (dict(half_extent=(1e300, 1.0, 0.2), step=(1e-300, 0.1, 0.02)), "params: more than 4194304 level-0 hypotheses"),
]


def _call(capi, lib, device, n=3, xyz=True, prior=True, params=True, out=True, n_out=True, cap=8, prior_value=None, **kw):
    p = dict(GOOD, **kw)
    prm = capi.PoseSearchParams((C.c_double * 3)(*p["half_extent"]), (C.c_double * 3)(*p["step"]), p["tau"], p["levels"], p["keep"])
    pts = np.zeros((min(max(n, 1), 16), 3))  # never read: every call here fails its checks first
    pr = np.array(prior_value if prior_value is not None else [0, 0, 0, 1.0, 0, 0, 0])
    o = (capi.PoseHypothesis * 64)()
    no, ns = C.c_int32(), C.c_int64()
    args = (C.byref(prm) if params else None, o if out else None, cap, C.byref(no) if n_out else None, C.byref(ns))
    if device:
        return lib.kicp_map_pose_search_device(None, pts.ctypes.data if xyz else None, n, capi.KICP_DTYPE_F64, 0, 0, 8, 16,
                                               capi.dp(pr) if prior else None, *args)
    return lib.kicp_map_pose_search(None, capi.dp(pts) if xyz else None, n, capi.dp(pr) if prior else None, *args)


@pytest.mark.parametrize("device", [False, True])
def test_validation(device):
    import __graft_entry__ as g
    g.build()
    from kinematic_icp_b200 import _capi
    lib = _capi.lib()
    fn = "kicp_map_pose_search_device" if device else "kicp_map_pose_search"

    def err(rc, text):
        assert rc == _capi.KICP_ERR_INVALID, rc
        msg = lib.kicp_last_error().decode()
        assert msg == "%s: %s" % (fn, text), msg

    err(_call(_capi, lib, device, n=-1), "n < 0")
    err(_call(_capi, lib, device, n=1 << 40), "n >= 2^30" if device else "n: 2^40 points or more")  # device clouds: < 2^30
    if not device:
        err(_call(_capi, lib, device, xyz=False), "xyz: null pointer")
    err(_call(_capi, lib, device, prior=False), "prior: null pointer")
    err(_call(_capi, lib, device, params=False), "params: null pointer")
    err(_call(_capi, lib, device, out=False), "out: null pointer")
    err(_call(_capi, lib, device, n_out=False), "n_out: null pointer")
    err(_call(_capi, lib, device, prior_value=[0, 0, 0, 1.0, float("nan"), 0, 0]), "prior: not finite")
    for kw, text in BAD:
        err(_call(_capi, lib, device, **kw), text)
    err(_call(_capi, lib, device, cap=7), "cap: below params->keep")
    err(_call(_capi, lib, device), "null map")


def test_python_keeps_host_and_device_arguments_apart():
    import kinematic_icp_b200 as kb
    m = kb.VoxelHashMap.__new__(kb.VoxelHashMap)
    with pytest.raises(ValueError):
        m.PoseSearch(np.zeros((3, 3)), np.r_[0, 0, 0, 1.0, 0, 0, 0], 0.5, (1, 1, 0.1), (0.1, 0.1, 0.1), point_step=20)
