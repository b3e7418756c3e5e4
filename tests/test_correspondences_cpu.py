"""The correspondence report without a GPU: kicp_corr_stats as gcc lays it out equals its ctypes mirrors, the new entry points reject
invalid arguments with KICP_ERR_INVALID before any device work (kicp_last_error names the argument)
and the Python layer keeps host and device arguments apart."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from corr_oracle import CorrStats
from kinematic_icp_b200._capi import KICP_DTYPE_F32 as F32, KICP_DTYPE_F64 as F64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    import __graft_entry__ as g
    g.build()
    from kinematic_icp_b200 import _capi
    return _capi, _capi.lib()


def test_corr_stats_layout_matches_header(tmp_path):
    """sizeof / offsetof of kicp_corr_stats (plain C) == the package's ctypes mirror == the tests' mirror; 80 bytes, no padding."""
    from kinematic_icp_b200 import _capi
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "kicp.h"', 'int main(void) {',
             'printf("sizeof %zu\\n", sizeof(kicp_corr_stats));']
    for fname, _ in _capi.CorrStats._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(kicp_corr_stats, %s));' % (fname, fname))
    lines += ['return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["sizeof"]) == C.sizeof(_capi.CorrStats) == C.sizeof(CorrStats) == 80
    for (fname, ftype), (tname, ttype) in zip(_capi.CorrStats._fields_, CorrStats._fields_):
        assert fname == tname and C.sizeof(ftype) == C.sizeof(ttype)
        assert int(out[fname]) == getattr(_capi.CorrStats, fname).offset == getattr(CorrStats, fname).offset, fname


def test_entry_points_reject_invalid_arguments_before_device_work():
    """One broken argument per call, a null map otherwise (checked after the arguments, before any device range): KICP_ERR_INVALID,
    with the call and the argument named.  No pointer is dereferenced."""
    _capi, L = _lib()
    INVALID = _capi.KICP_ERR_INVALID
    fake = 0x1000
    pose = np.array([0, 0, 0, 1.0, 0, 0, 0])
    pts = np.zeros((4, 3))
    dp = _capi.dp
    fn = b"kicp_map_correspondences"
    cases = [(lambda: L.kicp_map_correspondences(None, dp(pts), -1, dp(pose), 1.0, None, None, None, None), b"n < 0"),
             (lambda: L.kicp_map_correspondences(None, None, 4, dp(pose), 1.0, None, None, None, None), b"xyz: null pointer"),
             (lambda: L.kicp_map_correspondences(None, dp(pts), 4, None, 1.0, None, None, None, None), b"pose: null pointer"),
             (lambda: L.kicp_map_correspondences(None, dp(pts), 4, dp(pose), 1.0, None, None, None, None), b"null map")]
    for f, why in cases:
        assert f() == INVALID, why
        err = L.kicp_last_error()
        assert err.startswith(fn + b": ") and err.endswith(why), err
    fn = b"kicp_map_correspondences_device_async"
    good = dict(data=fake, n=4, dtype=F64, step=0, ox=0, oy=0, oz=0)
    broken = [({"n": -1}, b"n < 0"), ({"data": None}, b"data: null pointer"), ({"dtype": F32 + F64 + 7}, b"dtype"),
              ({"dtype": F32, "step": 12, "ox": 0, "oy": 4, "oz": 12}, b"point_step / offset"), ({}, b"null map")]
    for kw, why in broken:
        a = dict(good, **kw)
        c = (a["data"], a["n"], a["dtype"], a["step"], a["ox"], a["oy"], a["oz"])
        assert L.kicp_map_correspondences_device_async(None, *c, dp(pose), 1.0, fake, fake, fake, fake) == INVALID, kw
        err = L.kicp_last_error()
        assert err.startswith(fn + b": ") and why in err, (kw, err)
    c = (fake, 4, F64, 0, 0, 0, 0)
    assert L.kicp_map_correspondences_device_async(None, *c, None, 1.0, None, None, None, None) == INVALID
    assert L.kicp_last_error() == fn + b": pose: null pointer"
    # the frame's report: null arguments
    st = _capi.CorrStats()
    p = C.c_void_p()
    n = C.c_int64()
    for f, text in [(lambda: L.kicp_frame_correspondences(None, C.byref(st)), b"kicp_frame_correspondences: null context"),
                    (lambda: L.kicp_frame_correspondences(None, None), b"kicp_frame_correspondences: stats: null pointer"),
                    (lambda: L.kicp_frame_correspondences_device(None, C.byref(p), C.byref(p), C.byref(p), C.byref(n)),
                     b"kicp_frame_correspondences_device: null context"),
                    (lambda: L.kicp_frame_correspondences_device(None, None, C.byref(p), C.byref(p), C.byref(n)),
                     b"kicp_frame_correspondences_device: points: null pointer"),
                    (lambda: L.kicp_frame_correspondences_device(None, C.byref(p), None, C.byref(p), C.byref(n)),
                     b"kicp_frame_correspondences_device: dist: null pointer"),
                    (lambda: L.kicp_frame_correspondences_device(None, C.byref(p), C.byref(p), None, C.byref(n)),
                     b"kicp_frame_correspondences_device: inlier: null pointer"),
                    (lambda: L.kicp_frame_correspondences_device(None, C.byref(p), C.byref(p), C.byref(p), None),
                     b"kicp_frame_correspondences_device: n: null pointer")]:
        assert f() == INVALID, text
        assert L.kicp_last_error() == text


def test_option_is_declared_in_the_header():
    """The option is documented where kicp_ctx_set_option is, and the two frame readers are declared."""
    hdr = open(os.path.join(ROOT, "include", "kicp.h")).read()
    assert '"correspondences" 1 = every frame call' in hdr
    for name in ("kicp_frame_correspondences", "kicp_frame_correspondences_device", "kicp_map_correspondences_device_async"):
        assert name + "(" in hdr


def test_python_host_and_device_arguments_stay_apart(monkeypatch):
    """A host cloud takes none of the device keywords; a device cloud's out= must have the right shapes and types.  Checked before
    any call into the library (the map handle is a dummy)."""
    import kinematic_icp_b200 as kb
    from test_device_input_cpu import FakeArray

    m = kb.VoxelHashMap.__new__(kb.VoxelHashMap)
    m.h, m.ctx = None, None
    pose = np.array([0, 0, 0, 1.0, 0, 0, 0])
    with pytest.raises(ValueError, match="device inputs only"):
        m.Correspondences(np.zeros((3, 3)), pose, 1.0, stream=5)
    with pytest.raises(ValueError, match="device inputs only"):
        m.Correspondences(np.zeros((3, 3)), pose, 1.0, out=(1, 2, 3))
    dev = FakeArray((3, 3), "<f8", ptr=0x7F0000000000)
    with pytest.raises(ValueError, match="pass out="):
        m.Correspondences(dev, pose, 1.0)
    good = (FakeArray((3, 3), "<f8", ptr=0x7F0000001000), FakeArray((3,), "<f8", ptr=0x7F0000002000), FakeArray((3,), "|u1", ptr=0x7F0000003000))
    for k, bad in [(0, FakeArray((3, 3), "<f4", ptr=0x7F0000001000)), (1, FakeArray((4,), "<f8", ptr=0x7F0000002000)),
                   (2, FakeArray((3,), "<f8", ptr=0x7F0000003000))]:
        out = list(good)
        out[k] = bad
        with pytest.raises(ValueError, match=r"out\[%d\]" % k):
            m.Correspondences(dev, pose, 1.0, out=tuple(out))
