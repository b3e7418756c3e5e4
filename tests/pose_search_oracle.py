"""The pose search restated from the oracle (test infrastructure, shared by tests/test_pose_search_emu_cpu.py,
tests/test_pose_search_cpu.py and tests/test_gpu_pose_search.py): hypothesis poses with math.sin / math.cos in the operation order of
the facade's compat Eigen / Sophus, scores from ko.se3_transform and the oracle map's GetClosestNeighbor, the ranking key, the levels
and the merge.  sum_sq is also restated in k_pose_score's fixed summation order (kernel_sum), so the scores and therefore the
rankings are compared bit for bit."""
import ctypes as C
import math

import numpy as np

THREADS = 256  # k_pose_score's CTA: its summation order


class Params(C.Structure):
    """ctypes mirror of kicp_pose_search_params (include/kicp.h)"""
    _fields_ = [("half_extent", C.c_double * 3), ("step", C.c_double * 3), ("tau", C.c_double), ("levels", C.c_int32), ("keep", C.c_int32)]


class Hypothesis(C.Structure):
    """ctypes mirror of kicp_pose_hypothesis (include/kicp.h)"""
    _fields_ = [("pose", C.c_double * 7), ("offset", C.c_double * 3), ("lattice", C.c_int32 * 3), ("level", C.c_int32),
                ("n_inliers", C.c_int64), ("fitness", C.c_double), ("inlier_rmse", C.c_double), ("sum_sq", C.c_double)]


class Entry(C.Structure):
    """ctypes mirror of PsEntry (kicp_pose_search.h)"""
    _fields_ = [("L", C.c_int32 * 3), ("valid", C.c_int32), ("n_inl", C.c_int64), ("sum_sq", C.c_double)]


def params(half_extent, step, tau, levels, keep):
    return Params((C.c_double * 3)(*half_extent), (C.c_double * 3)(*step), tau, levels, keep)


def plan(half_extent, step, levels):
    """(k, scale, u): level-0 steps each side, finest steps per level-0 step, the finest steps"""
    scale = 2 ** (levels - 1)
    return [int(math.floor(half_extent[a] / step[a])) for a in range(3)], scale, [step[a] / scale for a in range(3)]


def rotation(prior, psi):
    """normalize(q_prior * (0, 0, sin(psi/2), cos(psi/2))) as (x, y, z, w)"""
    ax, ay, az, aw = (float(v) for v in prior[:4])
    bx, by, bz, bw = 0.0, 0.0, math.sin(psi / 2.0), math.cos(psi / 2.0)
    w = aw * bw - ax * bx - ay * by - az * bz
    x = aw * bx + ax * bw + ay * bz - az * by
    y = aw * by + ay * bw + az * bx - ax * bz
    z = aw * bz + az * bw + ax * by - ay * bx
    n2 = x * x
    n2 += y * y
    n2 += z * z
    n2 += w * w
    n = math.sqrt(n2)
    return [x / n, y / n, z / n, w / n]


def translation(prior, x, y):
    """t_prior + q_prior * (x, y, 0), quat_rotate's order"""
    qx, qy, qz, qw = (float(v) for v in prior[:4])
    px, py, pz = x, y, 0.0
    ux, uy, uz = qy * pz - qz * py, qz * px - qx * pz, qx * py - qy * px
    ux, uy, uz = ux + ux, uy + uy, uz + uz
    ox = px + qw * ux + (qy * uz - qz * uy)
    oy = py + qw * uy + (qz * ux - qx * uz)
    oz = pz + qw * uz + (qx * uy - qy * ux)
    return [float(prior[4]) + ox, float(prior[5]) + oy, float(prior[6]) + oz]


def pose(prior, u, L):
    """(pose7, offset) of lattice point L = (ix, iy, ipsi)"""
    off = [L[0] * u[0], L[1] * u[1], L[2] * u[2]]
    return np.array(rotation(prior, off[2]) + translation(prior, off[0], off[1])), off


def key(L, cnt, ssq):
    """the ranking key: more inliers, smaller sum_sq, smaller |ipsi|, smaller ix^2 + iy^2, then (ipsi, ix, iy)"""
    return (-cnt, ssq, abs(L[2]), L[0] * L[0] + L[1] * L[1], L[2], L[0], L[1])


def kernel_sum(v):
    """sum of v (float64, one value per point, 0 for non-inliers) in k_pose_score's order: thread t adds points t, t + 256, ... in
    turn; lane l of a warp adds threads l, l + 32, ..., l + 224; then the xor tree over the 32 lanes, read on lane 0"""
    v = np.asarray(v, dtype=np.float64)
    per = np.zeros(THREADS)
    if len(v):
        pad = np.zeros(-len(v) % THREADS)
        per = np.cumsum(np.concatenate([v, pad]).reshape(-1, THREADS), axis=0)[-1]
    lanes = np.zeros(32)
    for k in range(THREADS // 32):
        lanes = lanes + per[32 * k:32 * k + 32]
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[np.arange(32) ^ o]
    return float(lanes[0])


def score_many(ko, om, src, poses, tau):
    """[(n_inliers, kernel-order sum_sq, plain sum_sq)] of src at each pose"""
    src = np.ascontiguousarray(src, dtype=np.float64).reshape(-1, 3)
    n = len(src)
    if n == 0 or not len(poses):
        return [(0, 0.0, 0.0)] * len(poses)
    q = np.concatenate([ko.se3_transform(np.asarray(p, dtype=np.float64), src) for p in poses])
    _, d = om.nearest(q)
    out = []
    for h in range(len(poses)):
        dh = d[h * n:(h + 1) * n]
        inl = dh < tau
        dd = np.where(inl, dh, 0.0)
        sq = dd * dd
        out.append((int(inl.sum()), kernel_sum(sq), float(np.sum(sq[inl]))))
    return out


def search(ko, om, src, prior, tau, half_extent, step, levels, keep):
    """The search: returns dict(kept=[(L, n_inliers, sum_sq, level)] best first, scores={L: (n, sum_sq, plain, level)},
    level_kept=[set of L kept after each level], n_scored)"""
    k, scale, u = plan(half_extent, step, levels)
    prior = np.asarray(prior, dtype=np.float64)
    scores = {}

    def run(Ls, level):
        res = score_many(ko, om, src, [pose(prior, u, L)[0] for L in Ls], tau)
        for L, (c, s, p) in zip(Ls, res):
            scores[L] = (c, s, p, level)

    def best():
        return sorted(scores, key=lambda L: key(L, scores[L][0], scores[L][1]))[:keep]

    run([(ix * scale, iy * scale, ip * scale) for ip in range(-k[2], k[2] + 1) for ix in range(-k[0], k[0] + 1)
         for iy in range(-k[1], k[1] + 1)], 0)
    kept = best()
    level_kept = [list(kept)]
    for level in range(1, levels):
        s = 2 ** (levels - 1 - level)
        kids = []
        for c in kept:
            for dp in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    for dy in (-1, 0, 1):
                        L = (c[0] + dx * s, c[1] + dy * s, c[2] + dp * s)
                        if (dp or dx or dy) and L not in scores and L not in kids:
                            kids.append(L)
        run(kids, level)
        kept = best()
        level_kept.append(list(kept))
    return dict(kept=[(L, scores[L][0], scores[L][1], scores[L][3]) for L in kept], scores=scores, level_kept=level_kept,
                n_scored=len(scores), u=u)


def near_tie(res, rel=1e-9):
    """True when two scored hypotheses next to each other in the ranking around the kept boundary have equal counts and plain
    sums within rel (a ranking a different summation order could reorder)"""
    sc = res["scores"]
    order = sorted(sc, key=lambda L: key(L, sc[L][0], sc[L][2]))
    for a, b in zip(order, order[1:]):
        if sc[a][0] == sc[b][0] and abs(sc[a][2] - sc[b][2]) <= rel * max(abs(sc[a][2]), 1e-300) and sc[a][0] > 0:
            return True
    return False


def check_hypotheses(hyps, res, prior, n, rel=1e-12):
    """returned hypotheses (Hypothesis or PoseHypothesis-like with .lattice, .n_inliers, .sum_sq, .pose, .level) == the oracle's
    kept list: lattice points and levels in order, counts exactly, sum_sq bit for bit (kernel order) and within rel of the plain sum,
    pose bits"""
    want = res["kept"]
    assert len(hyps) == len(want), (len(hyps), len(want))
    for h, (L, c, s, level) in zip(hyps, want):
        assert tuple(h.lattice) == L, (tuple(h.lattice), L)
        assert h.n_inliers == c and h.level == level, (L, h.n_inliers, c, h.level, level)
        assert h.sum_sq == s, (L, h.sum_sq, s)
        plain = res["scores"][L][2]
        assert abs(h.sum_sq - plain) <= rel * abs(plain), (L, h.sum_sq, plain)
        p, off = pose(prior, res["u"], L)
        assert np.array_equal(np.asarray(h.pose, dtype=np.float64), p), (L, list(h.pose), p)
        assert list(h.offset) == off
        assert h.fitness == (c / n if n else 0.0)
        assert h.inlier_rmse == (math.sqrt(s / c) if c else 0.0)
