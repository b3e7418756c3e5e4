"""The oracles of the map queries at full size, checked on the CPU: the vectorised pose-search scorer (tests/map_query_batch_oracle.py)
against PO.score_many / PO.search on small lattices (ties, an empty map, non-finite points, n = 0, yaws at +-pi, several levels),
and AO.kernel_sum at 512 slots with more than one chunk per slot against a literal restatement of k_align_eval's loops."""
import math

import numpy as np

import align_planar_oracle as AO
import map_query_batch_oracle as BO
import pose_search_oracle as PO
import scenes as S


def _same_scores(ko, om, src, prior, tau, half_extent, step, levels, Ls):
    _, _, u = PO.plan(half_extent, step, levels)
    cnt, ssq, plain = BO.score(ko, om, src, prior, u, Ls, tau, max_queries=257)  # small batches: several per yaw
    want = PO.score_many(ko, om, src, [PO.pose(np.asarray(prior, dtype=np.float64), u, L)[0] for L in Ls], tau)
    for k, (c, s, p) in enumerate(want):
        assert cnt[k] == c and ssq[k] == s, (Ls[k], cnt[k], c, ssq[k], s)
        assert abs(plain[k] - p) <= 1e-13 * abs(p), (Ls[k], plain[k], p)
    return cnt


def _same_search(ko, om, src, prior, tau, half_extent, step, levels, keep):
    want = PO.search(ko, om, src, prior, tau, half_extent, step, levels, keep)
    got = BO.search(ko, om, src, prior, tau, half_extent, step, levels, keep)
    assert got["kept"] == want["kept"]
    assert got["level_kept"] == want["level_kept"]
    assert got["n_scored"] == want["n_scored"] and got["u"] == want["u"]
    for L, (c, s, p, level) in got["scores"].items():
        wc, ws, wp, wl = want["scores"][L]
        assert (c, s, level) == (wc, ws, wl) and abs(p - wp) <= 1e-13 * abs(wp), (L, c, s, p, level, want["scores"][L])
    return want


def test_quat_rotate_is_the_oracles_transform(oracle):
    """BO.quat_rotate + t is ko.se3_transform (the oracle's pose_apply) bit for bit"""
    ko = oracle
    rng = np.random.default_rng(1)
    pts = rng.normal(0, 30, (500, 3))
    for yaw in (0.0, 0.3, -math.pi, math.pi - 1e-3):
        T = ko.se3_compose(ko.planar_pose(4.2e5, 5.8e6, yaw), np.r_[rng.normal(size=4) * 0.01 + [0, 0, 0, 1], 0, 0, 0.5])
        T[:4] /= np.linalg.norm(T[:4])
        assert S.same_bits(BO.quat_rotate(T[:4], pts) + T[4:], ko.se3_transform(T, pts))


def test_kernel_sums_rows(oracle):
    rng = np.random.default_rng(2)
    for n in (0, 1, 31, 256, 257, 1000):
        v = rng.normal(size=(5, n)) * 10.0 ** rng.uniform(-8, 8, (5, n))
        assert S.same_bits(BO.kernel_sums(v), [PO.kernel_sum(r) for r in v])


def test_scores_on_ties_and_edges(oracle, workload):
    """every hypothesis of small lattices: the tie scenes, an empty map, non-finite points, n = 0, yaws at +-pi, cfg2"""
    ko = oracle
    for sc in S.tie_scenes(ko)[:3]:
        he, st = (0.25, 0.25, 0.1), (0.125, 0.125, 0.1)
        src = np.asarray(sc.scan, dtype=np.float64)[:60]
        Ls = [tuple(L) for L in BO.level0(he, st, 2)] + [(1, 3, -1), (-5, 2, 1)]
        _same_scores(ko, sc.om, src, ko.se3_compose(sc.last, sc.odom), sc.tau, he, st, 2, Ls)
    vs = 0.5
    rng = np.random.default_rng(8)
    pts = rng.uniform(-3, 3, (800, 3))
    om = ko.OracleMap(vs, S.FAR, 20)
    src = S.with_nonfinite(rng.uniform(-3, 3, (200, 3)), vs)
    he, st = (0.1, 0.1, 0.05), (0.05, 0.05, 0.05)
    Ls = [tuple(L) for L in BO.level0(he, st, 2)]
    assert not _same_scores(ko, om, src, ko.IDENTITY, 0.4, he, st, 2, Ls).any()
    om.add_points(pts)
    assert _same_scores(ko, om, src, ko.planar_pose(0.1, 0.05, 0.02), 0.4, he, st, 2, Ls).any()
    assert not _same_scores(ko, om, np.zeros((0, 3)), ko.IDENTITY, 0.4, he, st, 2, Ls).any()
    he, st = (0.0, 0.0, math.pi), (0.1, 0.1, math.pi / 4)
    _same_scores(ko, om, pts[:60], ko.planar_pose(0.0, 0.0, 3.0), 0.4, he, st, 2, [tuple(L) for L in BO.level0(he, st, 2)])
    w = workload(2)
    he, st = (0.2, 0.2, 0.04), (0.1, 0.1, 0.02)
    _same_scores(ko, w.map, w.scan[::97], w.prior, w.tau, he, st, 3, [tuple(L) for L in BO.level0(he, st, 3)])


def test_search_multi_level(oracle, workload):
    """the kept lists of every level, n_scored and the kept hypotheses' scores: cfg2 over three levels (keep 5 and 64), the tie
    scenes, the lattice of repeated patterns (score ties decided by the rest of the key), an empty map, non-finite points, n = 0
    and yaws at +-pi"""
    ko = oracle
    w = workload(2)
    src = w.scan[::max(1, len(w.scan) // 200)][:200]
    moved = ko.se3_compose(w.prior, ko.planar_pose(0.13, -0.07, 0.015))
    _same_search(ko, w.map, src, moved, w.tau, (0.2, 0.2, 0.04), (0.1, 0.1, 0.02), 3, 5)
    _same_search(ko, w.map, src[:40], moved, 0.3, (0.3, 0.3, 0.06), (0.1, 0.1, 0.02), 3, 64)
    for sc in S.tie_scenes(ko):
        src = np.asarray(sc.scan, dtype=np.float64)[:60]
        _same_search(ko, sc.om, src, ko.se3_compose(sc.last, sc.odom), sc.tau, (0.25, 0.25, 0.0), (0.125, 0.125, 0.1), 2, 6)
    grid = np.stack(np.meshgrid(np.arange(-4, 5), np.arange(-4, 5), [0.0], indexing="ij"), -1).reshape(-1, 3) + 0.5
    om = ko.OracleMap(1.0, S.FAR, 20)
    om.add_points(grid)
    res = _same_search(ko, om, grid[20:40], ko.IDENTITY, 0.3, (2.0, 2.0, 0.0), (1.0, 1.0, 0.1), 1, 8)
    assert len({(c, s) for _, c, s, _ in res["kept"]}) < len(res["kept"])
    vs = 0.5
    rng = np.random.default_rng(8)
    src = S.with_nonfinite(rng.uniform(-3, 3, (200, 3)), vs)
    _same_search(ko, ko.OracleMap(vs, S.FAR, 20), src, ko.IDENTITY, 1.0, (0.2, 0.2, 0.2), (0.1, 0.1, 0.1), 2, 7)
    pts = rng.uniform(-3, 3, (800, 3))
    om = ko.OracleMap(vs, S.FAR, 20)
    om.add_points(pts)
    _same_search(ko, om, src, ko.planar_pose(0.1, 0.05, 0.02), 0.4, (0.1, 0.1, 0.05), (0.05, 0.05, 0.05), 2, 4)
    _same_search(ko, om, np.zeros((0, 3)), ko.IDENTITY, 0.4, (0.1, 0.1, 0.1), (0.1, 0.1, 0.1), 2, 4)
    _same_search(ko, om, pts[:60], ko.planar_pose(0.0, 0.0, 3.0), 0.4, (0.0, 0.0, np.pi), (0.1, 0.1, np.pi / 4), 2, 5)


def _k_align_eval_sum(v, max_slots=512):
    """k_align_eval and k_align_step's order, loop by loop: slot c of C = min(max_slots, ceil(n / 256)) takes the chunks c, c + C,
    ...; lane j of warp w adds point 256 ch + 32 w + j of each; each warp's xor tree (o = 16 .. 1), read on lane 0; the warps added in
    index order; then the slots in index order"""
    n = len(v)
    chunks = (n + 255) // 256
    C = max(1, min(max_slots, chunks))
    total = 0.0
    for c in range(C):
        acc = [[0.0] * 32 for _ in range(8)]
        for ch in range(c, chunks, C):
            for w in range(8):
                for j in range(32):
                    i = 256 * ch + 32 * w + j
                    if i < n:
                        acc[w][j] += float(v[i])
        s = 0.0
        for w in range(8):
            lanes = acc[w]
            for o in (16, 8, 4, 2, 1):
                lanes = [lanes[j] + lanes[j ^ o] for j in range(32)]
            s += lanes[0]
        total += s
    return total


def test_align_kernel_sum_at_512_slots():
    """AO.kernel_sum at n = 131 072 (512 slots of one chunk), 131 073 (512 slots, slot 0 takes a second chunk of one point) and
    261 675 (cfg4's scan: 511 slots of two chunks and one of one, its last chunk 43 points) equals the restatement above bit for bit;
    with 256 slots the restatement gives other bits, so the slot count is visible in the sums"""
    rng = np.random.default_rng(5)
    differs = False
    for n in (131072, 131073, 261675):
        assert AO.slots(n) == 512 and (-(-n // 256) > 512) == (n > 131072)
        v = rng.normal(size=n) * 10.0 ** rng.uniform(-6, 6, n)
        v[rng.random(n) < 0.3] = 0.0
        want = _k_align_eval_sum(v)
        assert S.same_bits(AO.kernel_sum(v), want), n
        differs = differs or _k_align_eval_sum(v, 256) != want
    assert differs
