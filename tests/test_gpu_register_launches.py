"""The registration's launch sequence, entry point by entry point: kicp_register (packed float64), kicp_register_points (strided
float32 records) and kicp_register_scan_async (a device-resident scan; the result block pinned, pageable or NULL), each with the
options persistent 1 / 0, overlap_upload 1 / 0 and nn_cache 0 / 2.  The ctx.launch_count difference of every branch is pinned, and
so is what kicp_profile reports over the call.

Results: within one mode (persistent, nn_cache) every entry point gives the same iterations, status and per-pass correspondence
counts N, and the same pose and sums up to the order in which the kernel adds its per-CTA partial sums (which CTA takes which
window is decided at run time, so two runs of one registration may differ in the last bits of the sums); the float64 call matches
the CPU oracle as test_registration_configs_vs_oracle requires."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MAXIT = 10
TOL_T, TOL_R = 1e-6, 1e-7
EXPECTED = {
    # persistent 1: one cooperative launch of k_register runs the set-up and every pass
    "persistent: registration": 1,
    "persistent: n=0": 1,
    # persistent 0: k_reg_init, then k_register + k_solve for every pass, those issued after convergence included
    "per pass: registration": 1 + 2 * MAXIT,
    "per pass: n=0": 1 + 2 * MAXIT,
    # no pass to run: k_reg_init alone writes the prediction (Registration.cpp:157)
    "persistent: empty map": 1,
    "persistent: max_num_iterations=0": 1,
    "per pass: empty map": 1,
    "per pass: max_num_iterations=0": 1,
    # rejected before any device work
    "max_num_iterations > KICP_MAX_ITERATIONS": 0,
    "bad layout": 0,
    "sharded without a communicator": 0,
}
ENTRY_POINTS = ("kicp_register", "kicp_register_points", "scan_async pinned", "scan_async pageable", "scan_async NULL")


class Drive:
    """one context, its maps and the workload's scan; every call is recorded under its branch's name"""

    def __init__(self, kb, ctx, w, gm):
        from kinematic_icp_b200 import _capi
        self.kb, self.L, self.ctx, self.w, self.gm = kb, _capi.lib(), ctx, w, gm
        self.last, self.odom = _capi.as_pose(w.last_pose), _capi.as_pose(w.rel_odom)
        self.empty = kb.VoxelHashMap(ctx, w.voxel_size, w.max_range, w.max_points_per_voxel)
        self.launches, self.results = {}, {}
        self.pinned = kb.pinned_result()
        self.scan = kb.Scan(ctx)

    def close(self):
        self.L.kicp_host_free(C.addressof(self.pinned))
        self.scan.close()
        self.empty.close()

    def params(self, max_iter=MAXIT):
        return self.kb.RegParams(max_iter, 1, 1e-3, 0.0)

    def register(self, entry, gm, pts, params, sharded=False):
        """(status, result block or None) of one call; synchronises the context"""
        from kinematic_icp_b200._capi import KICP_DTYPE_F32, RegResult, dp
        L, w = self.L, self.w
        poses = (dp(self.last), dp(self.odom), w.tau, C.byref(params))
        out = np.empty(7)
        if entry == "kicp_register":
            res = RegResult()
            f = L.kicp_register_sharded if sharded else L.kicp_register
            return f(gm.h, dp(pts), len(pts), *poses, dp(out), C.byref(res)), res
        if entry == "kicp_register_points":  # 20-byte records: float32 intensity, then x, y, z
            rec = np.zeros((len(pts), 5), np.float32)
            rec[:, 1:4] = pts
            res = RegResult()
            f = L.kicp_register_points_sharded if sharded else L.kicp_register_points
            return f(gm.h, rec.ctypes.data, len(pts), KICP_DTYPE_F32, 20, 4, 8, 12, *poses, dp(out), C.byref(res)), res
        self.scan.upload(pts)
        res = {"scan_async pinned": self.pinned, "scan_async pageable": RegResult(), "scan_async NULL": None}[entry]
        f = L.kicp_register_scan_sharded_async if sharded else L.kicp_register_scan_async
        st = f(gm.h, self.scan.h, *poses, C.byref(res) if res is not None else None)
        self.ctx.synchronize()
        return st, res

    def call(self, name, entry, gm, pts, params, passes, sharded=False):
        """one call: its launches, and kicp_profile over it (`passes`: launches of k_register)"""
        self.ctx.profile_begin()
        l0 = self.ctx.launch_count
        st, res = self.register(entry, gm, pts, params, sharded)
        self.launches.setdefault(name, set()).add(self.ctx.launch_count - l0)
        prof = self.ctx.profile_end()
        if EXPECTED.get(name) == 0:
            assert st == 2 and prof.registrations == 0 and prof.assoc_launches + prof.idle_launches == 0, (name, entry, st)
            return None
        assert st in (0, 16), (name, entry, st)
        assert prof.registrations == 1 and prof.assoc_launches + prof.idle_launches == passes, (name, entry)
        return res, prof


def result_key(res):
    return (res.iterations, res.status, np.ctypeslib.as_array(res.sums)[: res.iterations, 5].tobytes())


def same_result(a, b):
    """same iterations, status and N; pose and sums up to the summation order of the per-CTA partial sums"""
    assert result_key(a) == result_key(b)
    assert np.allclose(a.pose_np(), b.pose_np(), rtol=0.0, atol=1e-12)
    assert np.allclose(a.sums_np(), b.sums_np(), rtol=1e-12, atol=1e-12)


def test_register_launches_per_entry_point(oracle, workload):
    import kinematic_icp_b200 as kb
    from test_gpu_parity import gpu_map_from_oracle
    w = workload(1)
    scan = np.ascontiguousarray(w.scan, np.float64)
    assert np.array_equal(scan.astype(np.float32).astype(np.float64), scan)  # the float32 records hold the very same scan
    po, ost = w.map.register(scan, w.last_pose, w.rel_odom, w.tau, max_iter=MAXIT)
    prediction = oracle.se3_compose(w.last_pose, w.rel_odom)
    ctx = kb.Context(0)
    gm = gpu_map_from_oracle(kb, ctx, w.map)
    d = Drive(kb, ctx, w, gm)
    try:
        for persistent in (1, 0):
            mode = "persistent" if persistent else "per pass"
            for overlap in (1, 0):
                for cache in (0, 2):
                    ctx.set_option("persistent", persistent)
                    ctx.set_option("overlap_upload", overlap)
                    ctx.set_option("nn_cache", cache)
                    for entry in ENTRY_POINTS:
                        res, prof = d.call(mode + ": registration", entry, gm, scan, d.params(), 1 if persistent else MAXIT)
                        if res is None:  # (the NULL result block: kicp_profile still reports the iteration count)
                            assert prof.assoc_iterations == ost.iterations
                            continue
                        assert prof.assoc_iterations == res.iterations == ost.iterations
                        assert prof.assoc_launches == (1 if persistent else res.iterations)
                        if not persistent:
                            assert prof.idle_launches == MAXIT - res.iterations > 0  # it converges early: idle passes
                        dt, ang = oracle.pose_delta(res.pose_np(), po)
                        assert dt <= TOL_T and ang <= TOL_R, (entry, dt, ang)
                        assert np.array_equal(res.sums_np()[:, 5], ost.sums_np()[:, 5])
                        assert np.allclose(res.sums_np()[:, :5], ost.sums_np()[:, :5], rtol=1e-9, atol=1e-9)
                        res = type(res).from_buffer_copy(res)
                        d.results.setdefault((persistent, cache), res)
                        same_result(d.results[(persistent, cache)], res)
                    for entry in ENTRY_POINTS:
                        res, prof = d.call(mode + ": n=0", entry, gm, scan[:0], d.params(), 1 if persistent else MAXIT)
                        assert res is None or res.iterations == prof.assoc_iterations
                        for name, m, params in (("empty map", d.empty, d.params()), ("max_num_iterations=0", gm, d.params(0))):
                            res, prof = d.call(mode + ": " + name, entry, m, scan, params, 0)
                            assert prof.assoc_iterations == 0
                            if res is not None:
                                assert res.iterations == 0
                                dt, ang = oracle.pose_delta(res.pose_np(), prediction)
                                assert dt < 1e-15 and ang < 1e-15, (name, entry)
        ctx.set_option("persistent", 1)
        for entry in ENTRY_POINTS:
            d.call("max_num_iterations > KICP_MAX_ITERATIONS", entry, gm, scan, d.params(65), 0)
            d.call("sharded without a communicator", entry, gm, scan, d.params(), 0, sharded=True)
        from kinematic_icp_b200._capi import KICP_DTYPE_F32, RegResult, dp
        ctx.profile_begin()
        l0 = ctx.launch_count
        rec = np.zeros((len(scan), 5), np.float32)
        out, res, params = np.empty(7), RegResult(), d.params()
        st = d.L.kicp_register_points(gm.h, rec.ctypes.data, len(scan), KICP_DTYPE_F32, 10, 0, 4, 8, dp(d.last), dp(d.odom), w.tau,
                                      C.byref(params), dp(out), C.byref(res))  # a point_step that is no multiple of 4
        d.launches.setdefault("bad layout", set()).add(ctx.launch_count - l0)
        assert st == 2 and ctx.profile_end().registrations == 0
        assert d.launches == {k: {v} for k, v in EXPECTED.items()}
    finally:
        d.close()
        gm.close()
        ctx.close()


def test_register_sharded_world_of_one(oracle, workload):
    """The sharded entry points over the peer exchange with one rank: the same launches and results as the unsharded calls"""
    import kinematic_icp_b200 as kb
    from test_gpu_parity import gpu_map_from_oracle
    w = workload(1)
    ctx = kb.Context(0)
    ctx.p2p_init([ctx.p2p_handle()], 1, 0)
    gm = gpu_map_from_oracle(kb, ctx, w.map)
    d = Drive(kb, ctx, w, gm)
    try:
        for cache in (0, 2):
            ctx.set_option("nn_cache", cache)
            ref = None
            for entry in ("kicp_register", "scan_async pinned", "scan_async pageable"):
                for sharded in (False, True):
                    res, prof = d.call("sharded world 1", entry, gm, w.scan, d.params(), 1, sharded=sharded)
                    assert prof.assoc_iterations == res.iterations and prof.assoc_launches == 1
                    res = type(res).from_buffer_copy(res)
                    ref = ref or res
                    same_result(ref, res)
        assert d.launches == {"sharded world 1": {1}}
    finally:
        d.close()
        gm.close()
        ctx.close()
