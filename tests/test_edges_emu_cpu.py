"""The map and front-end kernels at their decision boundaries, checked without a GPU: the scenes of tests/scenes.py ("edges") through
the emulated kernels (tests/emu), against the CPU oracle bit for bit.  Points exactly on voxel faces at voxel sizes that are not
powers of two, norms exactly equal to the range gate, candidates exactly map_resolution from a stored point, first points exactly
max_distance from the origin, probe chains of colliding keys that wrap past the last slot of the table, and NaN / +-Inf / huge
coordinates, whose voxel key is the one the reference gets on x86-64 (INT_MIN).  Floats are compared by bit pattern, so NaN equals
NaN.  The emulator compiles the kernels for x86, so it cannot see how the device converts a non-finite coordinate:
tests/test_gpu_edges.py runs the same scenes on the H100."""
import math

import numpy as np
import pytest

import scenes as S
from emu import harness as H
from test_kernel_emu_cpu import check as check_register

LAUNCHES = [(1, 1, 0), (2, 1, 1), (3, 0, 0), (3, 1, 1)]  # (grid, persistent, certificates)


def sorted_voxels(keys, counts, pts):
    off = np.concatenate([[0], np.cumsum(counts)])
    order = np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))
    return keys[order], counts[order], np.concatenate([pts[off[i]:off[i + 1]] for i in order]) if len(order) else pts


def assert_same_map(em, om):
    assert em.num_points() == om.num_points() and em.num_voxels() == om.num_voxels()
    k1, c1, p1 = sorted_voxels(*em.export_voxels())
    k0, c0, p0 = sorted_voxels(*om.export_voxels())
    assert np.array_equal(k1, k0) and np.array_equal(c1, c0) and S.same_bits(p1, p0)


def emu_map(vs, md, cap):
    return H.EmuMap(vs, md, cap, blocks_cap=4096)  # 16 384 slots: a table of the size the device starts with


# ---------------------------------------------------------------------------------------------------------- down-sample
def test_downsample_boundary_and_nonfinite_clouds(oracle):
    ko = oracle
    clouds = S.boundary_clouds()
    for vs, pts, flips, rounded in clouds:
        if vs in (0.37, 0.3, 0.1):  # the edge is there: quotients that round up onto an integer
            assert rounded > 0, vs
        for cloud in (pts, S.with_nonfinite(pts, vs)):
            ref = ko.voxel_downsample(cloud, vs)
            assert S.same_bits(H.downsample(cloud, vs), ref), vs
            # a stage of a frame: the count in a device word, a tail that must not be read
            n = len(cloud) - 7
            buf = np.concatenate([cloud[:n], np.full((7, 3), 1e6)])
            assert S.same_bits(H.downsample(buf, vs, n_actual=n), ko.voxel_downsample(cloud[:n], vs))
    # a reciprocal multiply would put these points into other voxels
    assert sum(f for vs, _, f, _ in clouds if vs in (0.37, 0.1)) > 20


def test_downsample_nan_first_in_voxel_zero(oracle):
    """A NaN point first in voxel (0, 0, 0) (under a conversion that gave 0 for NaN) must not replace that voxel's survivor."""
    ko = oracle
    for vs in (0.5, 0.37, 1.5):
        cloud = S.with_nonfinite(np.random.default_rng(3).uniform(-2, 2, (500, 3)) * vs, vs)
        ref = ko.voxel_downsample(cloud, vs)
        assert np.any(np.all(ref == 0.3 * vs, axis=1)), "the real point of voxel (0, 0, 0) survives in the reference"
        assert S.same_bits(H.downsample(cloud, vs), ref)


# ----------------------------------------------------------------------------------------------------------- Preprocess
@pytest.mark.parametrize("min_range,max_range", [(3.25, 104.0), (0.0, 13.0), (0.8125, 52.0)])
def test_preprocess_range_gate_exact_norms(oracle, min_range, max_range):
    ko = oracle
    pts, norms = S.range_gate_cloud(min_range if min_range else 13.0 / 16, max_range)
    assert (norms == max_range).sum() >= 7 and (norms < max_range).any() and (norms > max_range).any()
    if min_range:
        assert (norms == min_range).sum() >= 7
    pts = np.concatenate([pts, S.nonfinite_rows(1.0)])
    ref = ko.preprocess(pts, np.zeros(0), ko.IDENTITY, max_range, min_range, False)
    assert 0 < len(ref) < len(pts)
    assert S.same_bits(H.preprocess(ko, pts, np.zeros(0), ko.IDENTITY, max_range, min_range, False), ref)
    l2b = ko.se3_exp([0.2, -0.1, 0.3, 0.01, -0.02, 0.05])
    out = H.preprocess(ko, pts, np.zeros(0), ko.IDENTITY, max_range, min_range, False, lidar_to_base=l2b)
    assert S.same_bits(out, ko.se3_transform(l2b, ref))


def deskew_cases(ko):
    """(name, motion, stamps(n)) of the de-skew edges: pure translation (small-angle branch for every point), a rotation near pi and
    the same motion with a negative qw, a near-identity motion, every stamp equal (span 0: every point NaN, dropped), the extreme
    stamps at the first and the last index."""
    near_pi = ko.se3_exp([0.4, -0.2, 0.1, 0.0, 0.0, math.pi - 1e-3])
    neg = near_pi.copy()
    neg[:4] = -neg[:4]
    assert neg[3] < 0
    lin = lambda n: np.linspace(2.0, 2.1, n)
    ends = lambda n: np.r_[1.5, np.random.default_rng(1).uniform(1.6, 1.7, max(n - 2, 0)), 1.9][:n]
    return [("translation", ko.se3_exp([0.5, -0.3, 0.05, 0, 0, 0]), lin), ("near-pi", near_pi, lin), ("near-pi-negative-qw", neg, lin),
            ("near-identity", ko.se3_exp([1e-9, 0, 0, 1e-12, -1e-12, 1e-12]), lin), ("equal-stamps", ko.se3_exp([0.3, 0, 0, 0, 0, 0.1]),
             lambda n: np.full(n, 4.0)), ("extremes-first-last", ko.se3_exp([0.6, 0.02, 0.0, 0.001, -0.002, 0.03]), ends)]


def test_preprocess_deskew_edges(oracle, workload):
    ko = oracle
    w = workload(2)
    scan = np.concatenate([w.scan, w.scan, w.scan])  # several CTAs' shares of the stamps' min / max
    for name, motion, stamps_of in deskew_cases(ko):
        for pts in (scan, scan[:1]):
            stamps = stamps_of(len(pts))
            out = H.preprocess(ko, pts, stamps, motion, 100.0, 0.5, True)
            ref = ko.preprocess(pts, stamps, motion, 100.0, 0.5, True)
            assert out.shape == ref.shape, name
            if len(ref):
                assert np.abs(out - ref).max() < 1e-12, name
            if name == "equal-stamps" or len(pts) == 1:
                assert len(ref) == 0


# ------------------------------------------------------------------------------------------------------------------ map
@pytest.mark.parametrize("cap", [4, 16])
def test_addpoints_exact_map_resolution(oracle, cap):
    """Candidates exactly map_resolution from a stored point are kept (strict <), one ulp closer are dropped; voxels over-filled."""
    ko = oracle
    pts, exact, closer = S.map_rule_points(cap=cap)
    assert exact > 0 and closer > 0
    for seq in (pts, S.with_nonfinite(pts, 1.0)):
        om, em = ko.OracleMap(1.0, 100.0, cap), emu_map(1.0, 100.0, cap)
        try:
            om.add_points(seq)
            em.add_points(seq)
            assert_same_map(em, om)
            k, c, _ = om.export_voxels()
            assert np.any(c == cap) and np.any((c > 1) & (c < cap))
        finally:
            em.close()


@pytest.mark.parametrize("cap", [1, 255])
def test_addpoints_fills_extreme_caps(oracle, cap):
    """Caps 1 and 255 filled through AddPoints (pending lists longer than the replay's local array)."""
    ko = oracle
    rng = np.random.default_rng(cap)
    g = (np.stack(np.meshgrid(*[np.arange(7)] * 3, indexing="ij"), -1).reshape(-1, 3) + 0.5) / 7.0  # 343 points in one voxel
    pts = np.concatenate([(g[rng.permutation(len(g))] + [2, -3, 1]) * 0.37, rng.uniform(0, 4, (600, 3)) * 0.37,
                          S.with_nonfinite(rng.uniform(-1, 1, (300, 3)), 0.37)])
    om, em = ko.OracleMap(0.37, 100.0, cap), emu_map(0.37, 100.0, cap)
    try:
        for chunk in np.array_split(pts, 3):
            om.add_points(chunk)
            em.add_points(chunk)
        assert_same_map(em, om)
        assert om.export_voxels()[1].max() == cap
    finally:
        em.close()


def test_update_evicts_at_exactly_max_distance(oracle):
    """A voxel dies when its FIRST point is >= max_distance from the origin: exactly 12 away (144 exact) dies, one ulp inside lives,
    a far first point takes its near later points with it; a NaN first point never dies."""
    ko = oracle
    pts, sq = S.far_first_points()
    assert (sq == 144.0).any() and (sq < 144.0).any()
    for seq in (pts, S.with_nonfinite(pts, 3.0)):
        om, em = ko.OracleMap(3.0, 12.0, 8), emu_map(3.0, 12.0, 8)
        try:
            om.update_origin(seq, np.zeros(3))
            em.add_points(seq)
            em.remove_far(np.zeros(3))
            assert_same_map(em, om)
            assert om.num_voxels() < len(np.unique(np.floor(pts / 3.0), axis=0))  # something died
            om.update_pose(seq, ko.planar_pose(0.0, 0.0, 0.0))  # the asynchronous update: pose and count read on the device
            buf = np.concatenate([seq, np.full((5, 3), 1e9)])
            em.update_pose_async(buf, len(seq), ko.planar_pose(0.0, 0.0, 0.0))
            assert_same_map(em, om)
        finally:
            em.close()


def test_colliding_keys_wrap_the_table(oracle):
    """Voxels whose keys all share the last home slot: find-or-create and k_add_commit's own-slot search walk a chain that wraps
    past slot 0 (and collide inside one warp), k_nearest walks it to the end for absent keys."""
    ko = oracle
    keys = S.colliding_keys()
    for mask in (1023, 16383, (1 << 18) - 1):
        assert np.all(S.voxel_hash_np(*keys.T) & mask == mask)
    for sc in S.collision_scenes(ko):
        assert len(sc.present) >= 3
        # one AddPoints that creates every voxel of the chain at once, then a second that appends to them
        pts = sc.om.export_voxels()[2]
        om, em = ko.OracleMap(sc.voxel_size, S.FAR, sc.cap + 3), emu_map(sc.voxel_size, S.FAR, sc.cap + 3)
        try:
            om.add_points(pts[::2])
            em.add_points(pts[::2])
            om.add_points(np.concatenate([pts[1::2], S.with_nonfinite(sc.scan[:50], sc.voxel_size)]))
            em.add_points(np.concatenate([pts[1::2], S.with_nonfinite(sc.scan[:50], sc.voxel_size)]))
            assert_same_map(em, om)
            q = S.with_nonfinite(sc.scan, sc.voxel_size)
            pe, de = em.nearest(q)
            po, do = om.nearest(q)
            assert S.same_bits(de, do) and S.same_bits(pe, po), sc.name
            assert (do == np.finfo(np.float64).max).any()  # queries in absent colliding voxels found nothing
        finally:
            em.close()


def test_nearest_nonfinite_queries(oracle):
    """NaN, +-Inf and +-huge queries against a map that holds points under INT_MIN keys (-huge points): a +huge query must find
    them as the reference does."""
    ko = oracle
    vs = 0.5
    rng = np.random.default_rng(5)
    pts = np.concatenate([rng.uniform(-2, 2, (400, 3)), [[-3e9 * vs, 0.1, 0.1], [-3e9 * vs, -3e9 * vs, -3e9 * vs]]])
    om, em = ko.OracleMap(vs, 100.0, 20), emu_map(vs, 100.0, 20)
    try:
        om.add_points(pts)
        em.add_points(pts)
        assert_same_map(em, om)
        q = S.with_nonfinite(rng.uniform(-2, 2, (200, 3)), vs)
        pe, de = em.nearest(q)
        po, do = om.nearest(q)
        assert S.same_bits(de, do) and S.same_bits(pe, po)
        assert (do[np.all(q == 3e9 * vs, axis=1)] < np.finfo(np.float64).max).all()
    finally:
        em.close()


# --------------------------------------------------------------------------------------------------------- registration
@pytest.mark.parametrize("k", range(4), ids=["collide-3", "collide-9", "collide-17", "collide-40"])
def test_register_colliding_keys(emu_kr, oracle, k):
    """The registration kernel's probe of the home slot and the next one, its warp-uniform loop for longer chains (entered at
    h + 2) and the wrap, on maps whose every voxel sits in one chain; scan points in absent colliding voxels end their probe at an
    empty slot after the whole chain."""
    sc = S.collision_scenes(oracle)[k]
    for grid, persistent, cache in LAUNCHES:
        check_register(emu_kr, oracle, sc.om, sc.scan, sc.last, sc.odom, sc.tau, grid=grid, persistent=persistent, nn_cache=cache, **sc.kw)


def test_register_nonfinite_scan_points(emu_kr, oracle):
    """NaN, +-Inf and +-huge scan points have no correspondence in the reference; the kernel must drop them the same way."""
    sc = S.collision_scenes(oracle)[1]
    scan = S.with_nonfinite(sc.scan, sc.voxel_size)
    for grid, persistent, cache in LAUNCHES:
        check_register(emu_kr, oracle, sc.om, scan, sc.last, sc.odom, sc.tau, grid=grid, persistent=persistent, nn_cache=cache, max_iter=1)


@pytest.fixture(scope="module")
def emu_kr():
    return H.kr_lib()
