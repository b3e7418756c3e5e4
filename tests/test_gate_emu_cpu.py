"""The registration kernel's gate (Registration.cpp:75, (neighbor - query).norm() < tau) and its non-finite inputs, checked without a
GPU on the kernel emulator (tests/emu, tests/emu/variants.py) — built twice: "plain" (-ffp-contract=off: every unpinned expression in plain IEEE order, the
reference's) and "fma" (-mfma -ffp-contract=fast: the unpinned products and sums fused, as nvcc compiles kicp_register.cu).  A
decision that rests on an unpinned expression is the reference's in the plain build whatever the device does; only the contracting
build shows it.

The gate scenes of tests/gate_scenes.py put every query alone with one map point at a reference norm of exactly prev(tau), tau or
next(tau); at 20 or more of them per scene, each way of fusing the square would gate otherwise.  N of the first pass is defined bit
for bit: it must be the oracle's, and the count the scene makes itself.  The same build also runs the tie, shape and edge-case
registrations of test_kernel_emu_cpu.py."""
import math

import numpy as np
import pytest

import gate_scenes as G
import scenes as S
from emu import variants as V
from test_kernel_emu_cpu import TIE_IDS, SHAPE_IDS, TOL_R, TOL_T

VARIANTS = list(V.VARIANTS)
LAUNCHES = [(1, 1, 0), (2, 1, 1), (3, 0, 0), (2, 1, 0)]  # (grid, persistent, certificates): one per scene, in turn
GATE_IDS = ["tau0.05-vs0.5", "tau0.3-vs0.37-fixed", "tau1-vs1", "tau0.3-rotated", "tau0.3-far", "tau1-f32-fixed", "tau2.9-vs1",
            "dyadic", "dyadic-next"]
NONFINITE_IDS = ["vs0.75-cap24", "vs0.6-cap25", "tau1e12"]


@pytest.fixture(scope="module")
def gate_scenes(oracle):
    return G.gate_scenes(oracle)


@pytest.fixture(scope="module")
def nonfinite_scenes(oracle):
    return G.nonfinite_reg_scenes(oracle)


def check(ko, om, scan, last, odom, tau, **kw):
    """The checks of test_kernel_emu_cpu.check on the emulator of kw["variant"]: pose within the north-star tolerance, the same
    iteration count, N of every pass exactly, the sums to 1e-9, beta; every rank the same result."""
    res, stats = V.register(om, scan, last, odom, tau, **kw)
    okw = {k: kw[k] for k in ("max_iter", "conv", "adaptive", "fixed_reg") if k in kw}
    po, st = om.register(np.asarray(scan, dtype=np.float64), last, odom, tau, **okw)
    for r in res:
        dt, ang = ko.pose_delta(r.pose_np(), po)
        assert dt <= TOL_T and ang <= TOL_R, (dt, ang)
        assert r.iterations == st.iterations
        assert np.array_equal(r.sums_np()[:, 5], st.sums_np()[:, 5])
        assert np.allclose(r.sums_np()[:, :5], st.sums_np()[:, :5], rtol=1e-9, atol=1e-9)
        assert r.beta == pytest.approx(st.beta, rel=1e-10)
    for r in res[1:]:
        assert np.array_equal(r.pose_np(), res[0].pose_np()) and np.array_equal(r.sums_np(), res[0].sums_np())
    return res[0], stats


def launch(k):
    grid, persistent, cache = LAUNCHES[k % len(LAUNCHES)]
    return dict(grid=grid, persistent=persistent, nn_cache=cache)


# ------------------------------------------------------------------------------------------------------------ the scenes
def test_fast_fma_is_exact():
    """The scenes' FMA (math.fma or the C library's) is the exact, once-rounded a b + c."""
    rng = np.random.default_rng(1)
    for a, b, c in rng.normal(size=(2000, 3)) * [1.0, 1.0, 1e-3]:
        assert G.FMA(a, b, c) == S._fma(a, b, c)


@pytest.mark.parametrize("k", range(len(GATE_IDS)), ids=GATE_IDS)
def test_gate_scenes_keep_their_teeth(oracle, gate_scenes, k):
    """Each query's only candidate is the scene's point, at the reference norm the scene says; 20 or more points per contraction
    would be gated otherwise; the neighbour sits in the own voxel, a face, an edge or a corner voxel."""
    sc = gate_scenes[k]
    q = sc.queries(oracle)
    pts, d = sc.om.nearest(q)
    assert np.array_equal(pts, sc.cands)
    assert np.array_equal(d, [math.sqrt(S.ref_sq(c, x)) for c, x in zip(sc.cands, q)])
    assert sc.expected_n == int((d < sc.tau).sum())
    if sc.flips is None:  # the exact dyadic cases: every square is exact, nothing to flip
        assert all(not G.gate_flips(c, x, sc.tau) for c, x in zip(sc.cands, q))
        return
    assert min(sc.flips.values()) >= 20, sc.flips
    assert set(np.unique(d)) == {np.nextafter(sc.tau, 0.0), sc.tau, np.nextafter(sc.tau, np.inf)}
    if sc.tau < 0.5 * sc.voxel_size:
        assert min(sc.classes) > 0, sc.classes


# ------------------------------------------------------------------------------------------------------- the builds
def test_contracting_build_contracts_and_keeps_the_pinned_helpers(oracle, gate_scenes):
    """The "fma" build really fuses a plain a * b + c (a probe in the kernel's translation unit); dist2 and query_rn stay the
    reference's square and query in both builds."""
    sc = gate_scenes[0]
    q = sc.queries(oracle)
    trap = next(i for i, (c, x) in enumerate(zip(sc.cands, q)) if G.gate_flips(c, x, sc.tau))
    dx, dy = sc.cands[trap][0] - q[trap][0], sc.cands[trap][1] - q[trap][1]
    plain = dx * dx + dy * dy
    fused = G.FMA(dx, dx, dy * dy)
    assert plain != fused or G.FMA(dy, dy, dx * dx) != plain
    for variant in VARIANTS:
        L = V.kr_lib(variant)
        got = L.kr_emu_probe_fma(dx, dx, dy * dy)
        assert got == (fused if variant == "fma" else plain), variant
        prior = np.ascontiguousarray(oracle.se3_compose(sc.last, sc.odom))
        for c, x, p in zip(sc.cands, q, sc.scan):
            c, x, p = (np.ascontiguousarray(v, dtype=np.float64) for v in (c, x, p))
            assert L.kr_emu_dist2(c.ctypes.data, x.ctypes.data) == S.ref_sq(c, x), variant
            out = np.zeros(3)
            L.kr_emu_query(prior.ctypes.data, p.ctypes.data, out.ctypes.data)
            assert np.array_equal(out, x), variant
    rot = gate_scenes[3]  # and under a general rotation
    prior = np.ascontiguousarray(oracle.se3_compose(rot.last, rot.odom))
    for variant in VARIANTS:
        L = V.kr_lib(variant)
        for p, x in zip(rot.scan, rot.queries(oracle)):
            p, out = np.ascontiguousarray(p, dtype=np.float64), np.zeros(3)
            L.kr_emu_query(prior.ctypes.data, p.ctypes.data, out.ctypes.data)
            assert np.array_equal(out, x), variant


# ------------------------------------------------------------------------------------------------------- registrations
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("k", range(len(GATE_IDS)), ids=GATE_IDS)
def test_gate_matches_reference(emu_any, oracle, gate_scenes, k, variant):
    """The first pass gates every point as the reference does: N exactly the oracle's and the scene's own count, sums to 1e-9, the
    pose.  Every query's one candidate is evaluated, also at exactly tau (the search's bound min(best, tau^2) must not prune it)."""
    sc = gate_scenes[k]
    r, stats = check(oracle, sc.om, sc.scan, sc.last, sc.odom, sc.tau, variant=variant, **launch(k), **sc.kw)
    assert r.sums_np()[0, 5] == sc.expected_n
    assert stats[1] >= len(sc.scan)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("f32", [False, True], ids=["f64", "f32"])
@pytest.mark.parametrize("k", range(len(NONFINITE_IDS)), ids=NONFINITE_IDS)
def test_nonfinite_points_match_reference(emu_any, oracle, nonfinite_scenes, k, f32, variant):
    """NaN, +-Inf and +-3e9 vs scan points, and a map with non-finite points and voxels whose first point is NaN: N of every pass,
    no NaN in the sums, the pose.  tau = 1e12: the +huge queries are accepted against the INT_MIN voxel (N of the first pass and
    its sums only)."""
    sc = nonfinite_scenes[k]
    scan = sc.scan.astype(np.float32) if f32 else sc.scan
    lk = launch(k + 2 * f32)
    if k < 2:
        # (a +-3e9 vs point that finds its twin in a visible INT_MIN voxel is accepted: its Jacobian terms of 1e19 make the other
        # sums cancel, so they are held to 1e-9 of the largest sum of their pass)
        res, _ = V.register(sc.om, scan, sc.last, sc.odom, sc.tau, variant=variant, **lk, **sc.kw)
        po, st = sc.om.register(np.asarray(scan, dtype=np.float64), sc.last, sc.odom, sc.tau, **sc.kw)
        r = res[0]
        assert r.iterations == st.iterations
        got, want = r.sums_np()[:, :6], st.sums_np()[:, :6]
        assert np.array_equal(got[:, 5], want[:, 5])
        assert not np.isnan(got).any()
        scale = np.abs(want[:, :5]).max(axis=1, keepdims=True)
        assert np.all(np.abs(got[:, :5] - want[:, :5]) <= 1e-9 * scale)
        dt, ang = oracle.pose_delta(r.pose_np(), po)
        assert dt <= TOL_T and ang <= TOL_R, (dt, ang)
        return
    res, _ = V.register(sc.om, scan, sc.last, sc.odom, sc.tau, variant=variant, max_iter=1, **lk)
    _, st = sc.om.register(np.asarray(scan, dtype=np.float64), sc.last, sc.odom, sc.tau, max_iter=1)
    got, want = res[0].sums_np()[0], st.sums_np()[0]
    assert got[5] == want[5] and got[5] > 0
    assert not np.isnan(got).any()
    assert np.all(np.abs(got[:5] - want[:5]) <= 1e-9 * np.abs(want[:5]).max())


@pytest.fixture(scope="module")
def emu_any():
    for v in VARIANTS:
        V.kr_lib(v)


@pytest.fixture(scope="module")
def tie_scenes(oracle):
    return S.tie_scenes(oracle)


@pytest.fixture(scope="module")
def shape_scenes(oracle):
    return S.shape_scenes(oracle)


@pytest.mark.parametrize("k", range(len(TIE_IDS)), ids=TIE_IDS)
def test_neighbour_ties_under_contraction(emu_any, oracle, tie_scenes, k):
    """test_kernel_emu_cpu's tie scenes on the contracting build (one launch shape each)."""
    sc = tie_scenes[k]
    check(oracle, sc.om, sc.scan, sc.last, sc.odom, sc.tau, variant="fma", **launch(k), **sc.kw)


@pytest.mark.parametrize("k", range(len(SHAPE_IDS)), ids=SHAPE_IDS)
def test_map_shapes_under_contraction(emu_any, oracle, shape_scenes, k):
    sc = shape_scenes[k]
    check(oracle, sc.om, sc.scan, sc.last, sc.odom, sc.tau, variant="fma", **launch(k), **sc.kw)


def test_kernel_edge_cases_under_contraction(emu_any, oracle, workload):
    """test_kernel_emu_cpu's edge-case registrations on the contracting build."""
    from kinematic_icp_b200 import _capi
    ko = oracle
    w = workload(1)
    fma = dict(variant="fma")
    for n in (1, 31, 32, 33, 1000):
        check(ko, w.map, w.scan[:n], w.last_pose, w.rel_odom, w.tau, grid=2, **fma)
    check(ko, w.map, w.scan[:500], w.last_pose, w.rel_odom, w.tau, grid=2, nranks=2, **fma)
    res, _ = V.register(w.map, w.scan + 500.0, w.last_pose, w.rel_odom, w.tau, grid=2, **fma)
    assert np.all(np.isnan(res[0].pose_np())) and res[0].status == _capi.KICP_WARN_NO_CORRESPONDENCES
    check(ko, w.map, w.scan, w.last_pose, w.rel_odom, 0.3, grid=2, max_iter=1, **fma)
    check(ko, w.map, w.scan, w.last_pose, w.rel_odom, w.tau, grid=2, adaptive=False, fixed_reg=2.0, **fma)
    check(ko, w.map, w.scan, w.last_pose, w.rel_odom, w.tau, grid=3, conv=1e-6, max_iter=40, persistent=0, nn_cache=0, **fma)
    rng = np.random.default_rng(2)
    scan = w.scan + rng.normal(size=w.scan.shape) * 1e-3
    last = ko.se3_compose(w.last_pose, ko.se3_exp([0, 0, 0, 0.01, -0.02, 0.0]))
    r, _ = check(ko, w.map, scan, last, w.rel_odom, w.tau, grid=2, **fma)
    po, _ = w.map.register(scan, last, w.rel_odom, w.tau)
    dt, ang = ko.pose_delta(r.pose_np(), po)
    assert dt <= TOL_T and ang <= TOL_R
