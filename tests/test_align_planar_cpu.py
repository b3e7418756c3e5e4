"""The planar alignment without a GPU: the arithmetic the kernels, the emulator and the library share (kicp_align.h, through
tests/emu/kal_emu.cpp) bit for bit against the Python restatement (tests/align_planar_oracle.py) on random inputs; kicp_planar_align_params
and kicp_planar_alignment as gcc lays them out against their ctypes mirrors; and every argument check of kicp_map_align_planar* with its
text (the map is checked last, so each is reachable without a device)."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import align_planar_oracle as AO
from emu import harness as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _hooks():
    L = H.build("kal_emu")
    L.kal_update.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.kal_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.kal_step_norm.argtypes = [C.c_void_p]
    L.kal_step_norm.restype = C.c_double
    L.kal_align_slots.argtypes = [C.c_int64]
    return L


def test_update_bits():
    """T [+] dx from kicp_align.h == the restatement, bit for bit, and it turns by 2 atan(dx2 / 2)"""
    L = _hooks()
    rng = np.random.default_rng(5)
    for _ in range(300):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        T = np.ascontiguousarray(np.r_[q, rng.uniform(-500, 500, 3)])
        dx = np.ascontiguousarray(rng.normal(size=3) * 10.0 ** rng.integers(-12, 1))
        got = np.zeros(7)
        L.kal_update(T.ctypes.data, dx.ctypes.data, got.ctypes.data)
        assert np.array_equal(got, np.array(AO.update(T, dx))), (T, dx)
    T = np.ascontiguousarray([0, 0, 0, 1.0, 1.0, 2.0, 0.0])
    dx = np.ascontiguousarray([0.5, -0.25, 0.3])
    got = np.zeros(7)
    L.kal_update(T.ctypes.data, dx.ctypes.data, got.ctypes.data)
    assert abs(2 * math.atan2(got[2], got[3]) - 2 * math.atan(0.15)) < 1e-15 and list(got[4:]) == [1.5, 1.75, 0.0]


def test_solve_and_norm_bits():
    """the LDL^T solve and the step norm == the restatement, bit for bit: well-conditioned and near-singular systems, and the
    refusals (a zero, negative or non-finite pivot, a non-finite result)"""
    L = _hooks()
    rng = np.random.default_rng(6)
    cases = []
    for _ in range(300):
        J = rng.normal(size=(int(rng.integers(3, 9)), 3)) * rng.uniform(0.01, 100.0, 3)
        M = J.T @ J
        cases.append(([M[0, 0], M[0, 1], M[0, 2], M[1, 1], M[1, 2], M[2, 2]], rng.normal(size=3)))
    cases += [([1, 0, 0, 1, 0, 0], [1, 2, 3]), ([0, 0, 0, 1, 0, 1], [1, 1, 1]), ([-1, 0, 0, 1, 0, 1], [1, 1, 1]),
              ([1, 1, 0, 1, 0, 1], [1, 1, 1]), ([1, 0, 0, 1, 0, float("nan")], [1, 1, 1]), ([1, 0, 0, 1, 0, float("inf")], [1, 1, 1]),
              ([1e-300, 0, 0, 1, 0, 1], [1e300, 1, 1]), ([1, 0, 0, 1, 0, 1], [float("nan"), 0, 0]), ([4, 2, 2, 1, 1, 1], [1, 1, 1])]
    refused = 0
    for A, b in cases:
        A, b = np.ascontiguousarray(A, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
        dx = np.zeros(3)
        ok = L.kal_solve(A.ctypes.data, b.ctypes.data, dx.ctypes.data)
        want = AO.solve(A, b)
        assert ok == (want is not None), (A, b)
        if want is None:
            refused += 1
            continue
        assert list(dx) == want, (A, b, dx, want)
        assert L.kal_step_norm(dx.ctypes.data) == AO.step_norm(want)
    assert refused == 9  # every special case, no random system


def test_slots():
    L = _hooks()
    for n in (0, 1, 255, 256, 257, 600, 131072, 131073, 262144, 10 ** 7):
        assert L.kal_align_slots(n) == AO.slots(n)


def test_struct_layouts(tmp_path):
    """sizeof / offsetof of kicp_planar_align_params and kicp_planar_alignment (plain C) == the package's ctypes mirrors == the tests'"""
    from kinematic_icp_b200 import _capi
    pairs = {"kicp_planar_align_params": (_capi.PlanarAlignParams, AO.Params), "kicp_planar_alignment": (_capi.PlanarAlignment, AO.Alignment)}
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
    assert (_capi.KICP_ALIGN_CONVERGED, _capi.KICP_ALIGN_MAX_ITERATIONS, _capi.KICP_ALIGN_NO_CORRESPONDENCES,
            _capi.KICP_ALIGN_SINGULAR) == (AO.CONVERGED, AO.MAX_ITERATIONS, AO.NO_CORRESPONDENCES, AO.SINGULAR)


GOOD = dict(tau=0.5, convergence=1e-3, max_iterations=10)
BAD = [
    (dict(tau=float("nan")), "params->tau: not finite"),
    (dict(tau=float("inf")), "params->tau: not finite"),
    (dict(tau=0.0), "params->tau: not > 0"),
    (dict(tau=-1.0), "params->tau: not > 0"),
    (dict(convergence=float("nan")), "params->convergence: not finite"),
    (dict(convergence=-1e-9), "params->convergence: negative"),
    (dict(max_iterations=0), "params->max_iterations: not in 1..64"),
    (dict(max_iterations=65), "params->max_iterations: not in 1..64"),
]


def _call(capi, lib, device, n=3, xyz=True, initial=True, params=True, out=True, n_initial=2, start=None, **kw):
    p = dict(GOOD, **kw)
    prm = capi.PlanarAlignParams(p["tau"], p["convergence"], p["max_iterations"])
    pts = np.zeros((min(max(n, 1), 16), 3))  # never read: every call here fails its checks first
    starts = np.tile(np.array([0, 0, 0, 1.0, 0, 0, 0]), (65, 1))
    if start is not None:
        starts[1] = start
    o = (capi.PlanarAlignment * 65)()
    args = (capi.dp(starts) if initial else None, n_initial, C.byref(prm) if params else None, o if out else None)
    if device:
        return lib.kicp_map_align_planar_device(None, pts.ctypes.data if xyz else None, n, capi.KICP_DTYPE_F64, 0, 0, 8, 16, *args)
    return lib.kicp_map_align_planar(None, capi.dp(pts) if xyz else None, n, *args)


@pytest.mark.parametrize("device", [False, True])
def test_validation(device):
    import __graft_entry__ as g
    g.build()
    from kinematic_icp_b200 import _capi
    lib = _capi.lib()
    fn = "kicp_map_align_planar_device" if device else "kicp_map_align_planar"

    def err(rc, text):
        assert rc == _capi.KICP_ERR_INVALID, rc
        msg = lib.kicp_last_error().decode()
        assert msg == "%s: %s" % (fn, text), msg

    err(_call(_capi, lib, device, n=-1), "n < 0")
    err(_call(_capi, lib, device, n=1 << 40), "n >= 2^30" if device else "n: 2^40 points or more")  # device clouds: < 2^30
    if not device:
        err(_call(_capi, lib, device, xyz=False), "xyz: null pointer")
    err(_call(_capi, lib, device, initial=False), "initial: null pointer")
    err(_call(_capi, lib, device, params=False), "params: null pointer")
    err(_call(_capi, lib, device, out=False), "out: null pointer")
    for k in (0, -1, 65):
        err(_call(_capi, lib, device, n_initial=k), "n_initial: not in 1..64")
    for v in ([0, 0, 0, 1.0, float("nan"), 0, 0], [0, 0, float("inf"), 1.0, 0, 0, 0]):
        err(_call(_capi, lib, device, start=v), "initial: not finite")
    for kw, text in BAD:
        err(_call(_capi, lib, device, **kw), text)
    err(_call(_capi, lib, device, n_initial=64), "null map")
    err(_call(_capi, lib, device, n=0, xyz=False), "null map")


def test_python_arguments():
    import kinematic_icp_b200 as kb
    m = kb.VoxelHashMap.__new__(kb.VoxelHashMap)
    with pytest.raises(ValueError):
        m.AlignPlanar(np.zeros((3, 3)), np.r_[0, 0, 0, 1.0, 0, 0, 0], 0.5, point_step=20)
    with pytest.raises(ValueError):
        m.AlignPlanar(np.zeros((3, 3)), np.zeros((2, 6)), 0.5)
