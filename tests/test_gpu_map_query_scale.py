"""The map queries on the H100 at the sizes they are documented and benchmarked at (cfg4: a 1 001 499-point map at 0.5 m voxels and
its 261 675-point scan), where paths switch on that smaller calls never reach: k_align_eval with 512 slots of more than one chunk and a
64-start batch whose alignments stop at different iterations; k_pose_select over lists of lists (two and three rounds) and
k_pose_score grid-striding over more tiles than its resident grid, with refinement tiles spanning many rotations; k_pose_score with
about 1 000 points per thread; k_corr_eval on either side of every CTA-count boundary a resident grid of 1 to 4 CTAs per SM can have;
and the frame path's correspondence report at cfg4 size.  Each test first asserts that it reaches its path, by the host code's own
formulas, then compares with the oracles bit for bit (tests/align_planar_oracle.py, tests/map_query_batch_oracle.py,
tests/corr_oracle.py)."""
import numpy as np
import pytest

import align_planar_oracle as AO
import map_query_batch_oracle as BO
import pose_search_oracle as PO
from corr_oracle import check_stats, oracle_corr
from test_gpu_correspondences import st_c

pytestmark = pytest.mark.gpu
SMS = 132  # an H100 SXM's SMs
SELECT_ITEMS = 256 * 8  # k_pose_select: kPsThreads x kPsSelectItems items per CTA


def _map(kb, ctx, w):
    gm = kb.VoxelHashMap(ctx, w.voxel_size, w.max_range, w.max_points_per_voxel)
    gm.load_voxels(*w.map.export_voxels())
    return gm


def _cfg4(kb, workload):
    w = workload(4)
    assert len(w.scan) == 261675 and w.voxel_size == 0.5 and w.tau > w.voxel_size
    ctx = kb.Context(0)
    return w, ctx, _map(kb, ctx, w)


def select_rounds(n_hyp, keep):
    """k_pose_select's rounds over lists of lists after its first pass (ps_score_level's loop)"""
    rounds, items = 0, -(-n_hyp // SELECT_ITEMS) * keep
    while items > keep:
        items = -(-items // SELECT_ITEMS) * keep
        rounds += 1
    return rounds


@pytest.mark.parametrize("n", [261675, 131072, 131073, 196609])
def test_align_512_slots(oracle, workload, n):
    """the scan's first n points from the prior and two planar offsets of the true pose, at the registration's gate and at 0.3 m,
    bit for bit against AO.align.  n = 131 072 fills the 512 slots with one chunk each; above it slot c adds the chunks c, c + 512,
    ...: at 196 609 slot 0's second chunk is one point, at 261 675 slots 0-510 take two chunks and slot 511 one."""
    import kinematic_icp_b200 as kb
    ko = oracle
    chunks = -(-n // 256)
    if n == 131072:
        assert AO.slots(n) == 512 == chunks
    else:
        assert AO.slots(n) == 512 < chunks
    w, ctx, gm = _cfg4(kb, workload)
    try:
        src = np.ascontiguousarray(w.scan[:n])
        starts = np.array([w.prior, ko.se3_compose(w.true_pose, ko.planar_pose(0.13, -0.07, 0.015)),
                           ko.se3_compose(w.true_pose, ko.planar_pose(-0.05, 0.11, -0.02))])
        for tau in (w.tau, 0.3):
            got = gm.AlignPlanar(src, starts, tau)
            for k, (a, T0) in enumerate(zip(got, starts)):
                AO.check_alignment(a, AO.align(ko, w.map, src, T0, tau), (n, tau, k))
                assert a.n_inliers > n // 2
    finally:
        gm.close()
        ctx.close()


def test_align_batch_of_64_that_stop_apart(oracle, workload):
    """64 starts on the full scan, max_iterations 4, gate 0.3 m: near the true pose (CONVERGED within 2 iterations), 0.3 m / 0.03 rad
    off it (MAX_ITERATIONS) and 500 m away, outside the scene (NO_CORRESPONDENCES at once), interleaved, so that k_align_eval's
    32 768 blocks skip alignments that stopped at different iterations.  Every batched result is the same start alone bit for bit;
    one start of each kind is the oracle's."""
    import kinematic_icp_b200 as kb
    ko = oracle
    w, ctx, gm = _cfg4(kb, workload)
    try:
        src = np.ascontiguousarray(w.scan)
        rng = np.random.default_rng(64)
        kinds = [k % 3 for k in range(64)]
        starts = []
        for k in kinds:
            if k == 0:
                d = rng.uniform([-1e-3, -1e-3, -1e-4], [1e-3, 1e-3, 1e-4])
            elif k == 1:
                d = rng.uniform([0.25, -0.25, 0.025], [0.3, -0.2, 0.03])
            else:
                d = rng.uniform([490.0, 490.0, -0.1], [510.0, 510.0, 0.1])
            starts.append(ko.se3_compose(w.true_pose, ko.planar_pose(*d)))
        starts = np.array(starts)
        assert 64 * AO.slots(len(src)) == 32768
        many = gm.AlignPlanar(src, starts, 0.3, 4)
        want = {0: AO.CONVERGED, 1: AO.MAX_ITERATIONS, 2: AO.NO_CORRESPONDENCES}
        for k, (a, kind) in enumerate(zip(many, kinds)):
            one = gm.AlignPlanar(src, starts[k], 0.3, 4)[0]
            assert np.array_equal(one.pose, a.pose) and one[1:] == a[1:], k
            assert a.status == want[kind], (k, a.status)
            assert (a.iterations <= 2) if kind == 0 else (a.iterations == 4) if kind == 1 else (a.iterations == 0), (k, a.iterations)
        for k in (0, 1, 2):
            AO.check_alignment(many[k], AO.align(ko, w.map, src, starts[k], 0.3, 4), k)
    finally:
        gm.close()
        ctx.close()


def _few(w, n=24):
    return np.ascontiguousarray(w.scan[::len(w.scan) // n][:n])


def _search(ko, gm, om, src, prior, tau, he, st, levels, keep):
    hyps, n_scored = gm.PoseSearch(src, prior, tau, he, st, levels=levels, keep=keep)
    res = BO.search(ko, om, src, prior, tau, he, st, levels, keep)
    assert n_scored == res["n_scored"]
    PO.check_hypotheses(hyps, res, np.asarray(prior, dtype=np.float64), len(src))
    return res


@pytest.mark.parametrize("k, levels, rounds", [(20, 2, 2), (80, 1, 3)])
def test_pose_search_lists_of_lists(oracle, workload, k, levels, rounds):
    """keep 64 over a level 0 of (2k + 1)^3 hypotheses of 24 cfg4 points: 41^3 = 68 921 (two rounds of k_pose_select over lists of
    lists, then a refinement level) and 161^3 = 4 173 281 (three rounds, at the 4 194 304 limit); k_pose_score strides over more
    tiles than a resident grid of 4 CTAs per SM holds.  The kept list, counts, sums and poses against the vectorised oracle."""
    import kinematic_icp_b200 as kb
    ko = oracle
    st = (2.0 ** -4, 2.0 ** -4, 2.0 ** -7)
    he = tuple(k * s for s in st)
    kk, scale, _ = PO.plan(he, st, levels)
    assert kk == [k, k, k]
    n0 = (2 * k + 1) ** 3
    assert n0 <= 4194304 and select_rounds(n0, 64) == rounds
    assert (2 * k + 1) * -(-(2 * k + 1) ** 2 // 8) > 4 * SMS
    w, ctx, gm = _cfg4(kb, workload)
    try:
        prior = ko.se3_compose(w.true_pose, ko.planar_pose(0.4, -0.3, -0.15))  # the true yaw near +19 steps: late in level 0
        res = _search(ko, gm, w.map, _few(w), prior, 0.3, he, st, levels, 64)
        assert res["kept"][0][1] > 0 and len(res["kept"]) == 64
        # round r's first CTA selects from the first 32^r x 2048 hypotheses (32 lists of 64 per CTA); a kept level-0 hypothesis
        # beyond them is missed by a search that stops after round r < rounds
        n = 2 * k + 1
        h = [((L[2] // scale + k) * n + L[0] // scale + k) * n + L[1] // scale + k for L, _, _, level in res["kept"] if level == 0]
        for r in range(1, rounds):
            assert max(h) >= 32 ** r * SELECT_ITEMS, (r, max(h))
    finally:
        gm.close()
        ctx.close()


def test_pose_search_refinement_over_many_rotations(oracle, workload):
    """keep 64 over 3 levels on cfg2, with yaw steps small enough that the 64 parents of a refinement level lie on many rotations,
    so its tiles mix them"""
    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(2)
    ctx = kb.Context(0)
    gm = _map(kb, ctx, w)
    try:
        src = np.ascontiguousarray(w.scan[::len(w.scan) // 300][:300])
        prior = ko.se3_compose(w.true_pose, ko.planar_pose(0.21, 0.13, -0.03))
        res = _search(ko, gm, w.map, src, prior, 0.3, (0.4, 0.4, 0.008), (0.1, 0.1, 0.002), 3, 64)
        assert len({L[2] for L in res["level_kept"][0]}) >= 5 and len({L[2] for L in res["level_kept"][1]}) >= 5
        assert res["n_scored"] > 9 ** 3 + 2 * 64
    finally:
        gm.close()
        ctx.close()


def test_pose_search_many_points_per_thread(oracle, workload):
    """the full cfg4 scan on a 3 x 3 x 3 level 0 (each thread of k_pose_score evaluates 1 022 or 1 023 points per hypothesis),
    every hypothesis against the vectorised oracle"""
    import kinematic_icp_b200 as kb
    ko = oracle
    w, ctx, gm = _cfg4(kb, workload)
    try:
        src = np.ascontiguousarray(w.scan)
        assert -(-len(src) // 256) == 1023
        prior = ko.se3_compose(w.true_pose, ko.planar_pose(0.05, -0.03, 0.01))
        res = _search(ko, gm, w.map, src, prior, w.tau, (0.1, 0.1, 0.01), (0.1, 0.1, 0.01), 1, 27)
        assert res["n_scored"] == 27 and res["kept"][0][1] > res["kept"][-1][1]
    finally:
        gm.close()
        ctx.close()


def test_correspondences_cfg4(oracle, workload):
    """the full scan at the prior and at a planar offset: per-point outputs bit for bit against the oracle; then prefixes of n =
    8 k 132 - 1, + 0 and + 1 (k = 1..4): k_corr_eval's grid min(ceil(n / 8), resident) crosses k CTAs per SM of 132 SMs there"""
    import kinematic_icp_b200 as kb
    ko = oracle
    w, ctx, gm = _cfg4(kb, workload)
    try:
        src = np.ascontiguousarray(w.scan)
        for pose in (w.prior, ko.se3_compose(w.true_pose, ko.planar_pose(0.3, -0.2, 0.02))):
            po, do, io, want = oracle_corr(ko, w.map, src, pose, w.tau)
            p, d, inl, st = gm.Correspondences(src, pose, w.tau)
            assert np.array_equal(d.view(np.uint64), do.view(np.uint64)) and np.array_equal(p.view(np.uint64), po.view(np.uint64))
            assert np.array_equal(inl.astype(bool), io)
            check_stats(st_c(st), want)
            assert 0 < want["n_inliers"] < len(src)
        for k in range(1, 5):
            for n in (8 * k * SMS - 1, 8 * k * SMS, 8 * k * SMS + 1):
                assert -(-n // 8) == k * SMS + (n > 8 * k * SMS)
                *_, want = oracle_corr(ko, w.map, src[:n], w.prior, w.tau)
                *_, st = gm.Correspondences(src[:n], w.prior, w.tau)
                check_stats(st_c(st), want)
    finally:
        gm.close()
        ctx.close()


@pytest.mark.parametrize("gated", [False, True])
def test_frame_report_cfg4(oracle, workload, gated):
    """one kicp_register_frame of the cfg4 scan with option "correspondences" 1 (and the GATED map update): the frame's report is
    Correspondences of the returned source at the returned pose against the map before the frame's Update, taken with
    export_voxels beforehand; the report's count lives in device memory and the host bound is the frame's size, several times
    larger"""
    import torch

    import kinematic_icp_b200 as kb
    ko = oracle
    w, ctx, gm = _cfg4(kb, workload)
    ref = None
    try:
        ctx.set_option("correspondences", 1)
        if gated:
            ctx.set_map_update(kb._capi.KICP_MAP_UPDATE_GATED, min_inliers=1000, min_fitness=0.5, max_inlier_rmse=1.0)
        before = gm.export_voxels()
        ident = np.ascontiguousarray(ko.IDENTITY)
        pose, _, source, _ = kb.RegisterFrame(gm, w.scan, np.zeros(0), ident, ident, w.last_pose, w.rel_odom, w.tau, max_range=100.0,
                                              min_range=0.0, deskew=False, voxel_size=w.voxel_size)
        source = np.ascontiguousarray(source, dtype=np.float64)
        assert 0 < 2 * len(source) < len(w.scan)
        if gated:
            assert kb.frame_map_update(ctx) == kb._capi.KICP_FRAME_UPDATE_APPLIED
        pts, dist, inl = (torch.as_tensor(a, device="cuda").cpu().numpy() for a in kb.frame_correspondences_device(ctx))
        st = kb.frame_correspondences(ctx)
        ref = kb.VoxelHashMap(ctx, w.voxel_size, w.max_range, w.max_points_per_voxel)
        ref.load_voxels(*before)
        rp, rd, ri, rst = ref.Correspondences(source, pose, w.tau)
        assert np.array_equal(dist.view(np.uint64), rd.view(np.uint64)) and np.array_equal(pts.view(np.uint64), rp.view(np.uint64))
        assert np.array_equal(inl, ri)
        assert st.n_points == rst.n_points == len(source) and st.n_inliers == rst.n_inliers > len(source) // 2
        om = ko.OracleMap(w.voxel_size, w.max_range, w.max_points_per_voxel)
        om.add_points(before[2])
        po, do, io, want = oracle_corr(ko, om, source, pose, w.tau)
        assert np.array_equal(dist.view(np.uint64), do.view(np.uint64)) and np.array_equal(inl.astype(bool), io)
        check_stats(st_c(st), want)
        check_stats(st_c(rst), want)
    finally:
        if ref is not None:
            ref.close()
        gm.close()
        ctx.close()
