"""The registration kernel's emulator (tests/emu/kr_emu.cpp) in two builds (test infrastructure).

"plain" is g++ -ffp-contract=off, as harness.kr_lib() builds it: every unpinned expression in plain IEEE order (the reference's).
"fma" is -O2 -mfma -ffp-contract=fast: the unpinned products and sums fused, as nvcc compiles kicp_register.cu (GCC contracts only
at -O2 and above), so an exact decision that rests on an unpinned expression shows there.  Both compile kr_emu_variants.cpp, where
the pinned helpers (__dmul_rn, add_rn) stay unfused.  The map and front-end emulators are built plain only: their kernels are built -fmad=false."""
import ctypes as C
import os
import subprocess

import numpy as np

from emu import harness as H

FLAGS = {"plain": ["-O1", "-ffp-contract=off"], "fma": ["-O2", "-mfma", "-ffp-contract=fast"]}
VARIANTS = tuple(FLAGS)
_LIBS = {}


def kr_lib(variant="plain"):
    """The registration emulator of `variant` (kr_emu_variants.cpp), with the self-check entry points typed."""
    if variant not in _LIBS:
        out = os.path.join(H.EMU, "_build")
        os.makedirs(out, exist_ok=True)
        so = os.path.join(out, "libkr_emu_%s.so" % variant)
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++"] + FLAGS[variant] + ["-std=c++17", "-fPIC", "-shared", "-I" + cuda_inc, "-I" + os.path.join(H.ROOT, "include"),
                        "-I" + os.path.join(H.ROOT, "kinematic-icp_b200", "csrc"), "-o", so, os.path.join(H.EMU, "kr_emu_variants.cpp"),
                        "-lpthread"], check=True)
        L = C.CDLL(so)
        L.kr_emu_probe_fma.restype = C.c_double
        L.kr_emu_probe_fma.argtypes = [C.c_double, C.c_double, C.c_double]
        L.kr_emu_dist2.restype = C.c_double
        L.kr_emu_dist2.argtypes = [C.c_void_p, C.c_void_p]
        L.kr_emu_query.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _LIBS[variant] = L
    return _LIBS[variant]


def register(om, scan, last, odom, tau, variant="plain", grid=3, nranks=1, persistent=1, nn_cache=1, registrations=1, max_iter=10,
             conv=1e-3, adaptive=True, fixed_reg=0.0):
    """harness.register on the emulator of `variant`: ([RegResult per rank], [probes, candidate points, lines])."""
    from kinematic_icp_b200 import _capi
    lib = kr_lib(variant)
    keys, counts, pts = om.export_voxels()
    keys = np.ascontiguousarray(keys, dtype=np.int32)
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    pts = np.ascontiguousarray(pts, dtype=np.float64)
    f32 = scan.dtype == np.float32
    scan = np.ascontiguousarray(scan)
    last, odom = np.ascontiguousarray(last, dtype=np.float64), np.ascontiguousarray(odom, dtype=np.float64)
    p = _capi.RegParams(max_iter, 1 if adaptive else 0, conv, fixed_reg)
    res = (_capi.RegResult * nranks)()
    stats = (C.c_uint64 * 3)()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib.kr_emu_register(vp(keys), vp(counts), vp(pts), C.c_int64(len(counts)), C.c_int32(om.max_points_per_voxel),
                             C.c_double(om.voxel_size), vp(scan), C.c_int64(len(scan)), C.c_int32(1 if f32 else 0), vp(last), vp(odom),
                             C.c_double(tau), C.byref(p), C.c_int32(grid), C.c_int32(nranks), C.c_int32(persistent), C.c_int32(nn_cache),
                             C.c_int32(registrations), res, stats, C.c_int32(0), C.c_int32(-1))
    assert rc == 0, "a launch must leave its counters zero for the next one: rc %d" % rc
    return list(res), list(stats)
