"""The correspondence report composed from the oracle (test infrastructure, shared by tests/test_correspondences_emu_cpu.py and
tests/test_gpu_correspondences.py): the oracle's T * p, the oracle's GetClosestNeighbor of it, the gate d < tau, and
ComputePerturbation's Jacobian and residual (Registration.cpp:89-95) in numpy."""
import ctypes as C

import numpy as np


class CorrStats(C.Structure):
    """ctypes mirror of kicp_corr_stats (include/kicp.h)."""
    _fields_ = [("n_points", C.c_int64), ("n_inliers", C.c_int64), ("fitness", C.c_double), ("inlier_rmse", C.c_double),
                ("sum_sq", C.c_double), ("jtj", C.c_double * 3), ("jtr", C.c_double * 2)]

    def sums(self):
        """[sum_sq, JTJ00, JTJ01, JTJ11, JTr0, JTr1]"""
        return np.array([self.sum_sq, *self.jtj, *self.jtr])


def oracle_corr(ko, om, src, pose, tau):
    """(points, dist, inlier, dict of the statistics) of `src` at `pose` against the oracle map `om`."""
    src = np.ascontiguousarray(src, dtype=np.float64).reshape(-1, 3)
    pose = np.ascontiguousarray(pose, dtype=np.float64)
    n = len(src)
    if n == 0:
        return np.zeros((0, 3)), np.zeros(0), np.zeros(0, bool), dict(n_points=0, n_inliers=0, fitness=0.0, inlier_rmse=0.0,
                                                                       sums=np.zeros(6), scale=np.zeros(6))
    q = ko.se3_transform(pose, src)
    nb, d = om.nearest(q)
    inl = d < tau
    rot = np.r_[pose[:4], 0.0, 0.0, 0.0]
    s, p = src[inl], q[inl]
    r = p - nb[inl]
    a = ko.se3_transform(rot, np.tile([1.0, 0.0, 0.0], (max(len(s), 1), 1)))[: len(s)]
    b = ko.se3_transform(rot, np.stack([-s[:, 1], s[:, 0], np.zeros(len(s))], 1)) if len(s) else np.zeros((0, 3))
    terms = [r * r, a * a, a * b, b * b, a * r, b * r]
    sums = np.array([t.sum() for t in terms])
    k = int(inl.sum())
    stats = dict(n_points=n, n_inliers=k, fitness=k / n, inlier_rmse=float(np.sqrt(sums[0] / k)) if k else 0.0, sums=sums,
                 scale=np.array([np.abs(t).sum() for t in terms]))
    return nb, d, inl, stats


def close_sums(got, want, scale, rel=1e-12):
    """every sum within rel of the oracle's, relative to the sum of its terms' magnitudes (a signed sum such as JTr may cancel to
    near 0, where only the summation order separates two correct results)"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return bool(np.all(np.abs(got - want) <= rel * np.asarray(scale))), (got, want)


def check_stats(st, want, rel=1e-12):
    """a kicp_corr_stats (CorrStats) against oracle_corr's statistics: the counts exactly, the sums to `rel`"""
    assert st.n_points == want["n_points"] and st.n_inliers == want["n_inliers"], (st.n_points, st.n_inliers, want)
    k, n = want["n_inliers"], want["n_points"]
    assert st.fitness == (k / n if n else 0.0)
    ok, info = close_sums(st.sums(), want["sums"], want["scale"], rel)
    assert ok, info
    if k:
        assert abs(st.inlier_rmse - want["inlier_rmse"]) <= rel * want["inlier_rmse"] + 1e-300
    else:
        assert st.inlier_rmse == 0.0 and not st.sums().any()
