"""The planar alignment restated from the oracle (test infrastructure, shared by tests/test_align_planar_emu_cpu.py,
tests/test_align_planar_cpu.py and tests/test_gpu_align_planar.py): query points from ko.se3_transform, neighbours and distances from
the oracle map's GetClosestNeighbor, the Jacobian and the sums in k_align_eval's operation order and fixed summation order, the LDL^T
solve, the update T [+] dx (no trigonometry) and the stopping rules of kicp_align.h, all in float64 with one rounding per operation.
Every iteration's pose, the status, the iteration count and the report at the returned pose therefore compare bit for bit."""
import ctypes as C
import math

import numpy as np

THREADS = 256  # k_align_eval's CTA: 8 warps, one 256-point chunk at a time
MAX_SLOTS = 512  # kAlignCtas
DBL_MAX = np.finfo(np.float64).max
CONVERGED, MAX_ITERATIONS, NO_CORRESPONDENCES, SINGULAR = 0, 1, 2, 3


class Params(C.Structure):
    """ctypes mirror of kicp_planar_align_params (include/kicp.h)"""
    _fields_ = [("tau", C.c_double), ("convergence", C.c_double), ("max_iterations", C.c_int32)]


class Alignment(C.Structure):
    """ctypes mirror of kicp_planar_alignment (include/kicp.h)"""
    _fields_ = [("pose", C.c_double * 7), ("status", C.c_int32), ("iterations", C.c_int32), ("last_step", C.c_double),
                ("n_inliers", C.c_int64), ("fitness", C.c_double), ("inlier_rmse", C.c_double), ("sum_sq", C.c_double),
                ("jtj", C.c_double * 6), ("jtr", C.c_double * 3)]


def slots(n):
    """CTA slots of one alignment: min(kAlignCtas, ceil(n / 256)), at least 1"""
    return min(MAX_SLOTS, max(1, -(-n // THREADS)))


def update(T, dx):
    """T [+] dx: normalize(q_T * (0, 0, dx2 / 2, 1)), t_T + R_T (dx0, dx1, 0), kicp_align.h's operation order"""
    ax, ay, az, aw = (float(v) for v in T[:4])
    bx, by, bz, bw = 0.0, 0.0, float(dx[2]) / 2.0, 1.0
    w = aw * bw - ax * bx - ay * by - az * bz
    x = aw * bx + ax * bw + ay * bz - az * by
    y = aw * by + ay * bw + az * bx - ax * bz
    z = aw * bz + az * bw + ax * by - ay * bx
    n2 = x * x
    n2 += y * y
    n2 += z * z
    n2 += w * w
    ln = math.sqrt(n2)
    px, py, pz = float(dx[0]), float(dx[1]), 0.0
    ux, uy, uz = ay * pz - az * py, az * px - ax * pz, ax * py - ay * px
    ux, uy, uz = ux + ux, uy + uy, uz + uz
    ox = px + aw * ux + (ay * uz - az * uy)
    oy = py + aw * uy + (az * ux - ax * uz)
    oz = pz + aw * uz + (ax * uy - ay * ux)
    return [x / ln, y / ln, z / ln, w / ln, float(T[4]) + ox, float(T[5]) + oy, float(T[6]) + oz]


def _pivot_ok(d):
    return d > 0.0 and d <= DBL_MAX


def solve(A, b):
    """dx = -A^-1 b by kicp_align.h's fixed LDL^T, A = (a00, a01, a02, a11, a12, a22); None when a pivot is not positive and finite
    or dx is not finite"""
    A = [float(v) for v in A]
    b = [float(v) for v in b]
    d0 = A[0]
    if not _pivot_ok(d0):
        return None
    l10, l20 = A[1] / d0, A[2] / d0
    d1 = A[3] - l10 * A[1]
    if not _pivot_ok(d1):
        return None
    e = A[4] - l20 * A[1]
    l21 = e / d1
    d2 = (A[5] - l20 * A[2]) - l21 * e
    if not _pivot_ok(d2):
        return None
    y0 = -b[0]
    y1 = -b[1] - l10 * y0
    y2 = (-b[2] - l20 * y0) - l21 * y1
    z0, z1, z2 = y0 / d0, y1 / d1, y2 / d2
    x2 = z2
    x1 = z1 - l21 * x2
    x0 = (z0 - l10 * x1) - l20 * x2
    dx = [x0, x1, x2]
    return dx if all(math.isfinite(v) for v in dx) else None


def step_norm(dx):
    return math.sqrt((dx[0] * dx[0] + dx[1] * dx[1]) + dx[2] * dx[2])


def _quat_rotate(qx, qy, qz, qw, px, py, pz):
    ux, uy, uz = qy * pz - qz * py, qz * px - qx * pz, qx * py - qy * px
    ux, uy, uz = ux + ux, uy + uy, uz + uz
    return px + qw * ux + (qy * uz - qz * uy), py + qw * uy + (qz * ux - qx * uz), pz + qw * uz + (qx * uy - qy * ux)


def kernel_sum(v):
    """sum of v (one float64 per point, 0 for non-inliers) in k_align_eval's order: slot c of C adds the 256-point chunks c, c + C,
    ... lane by lane (point 32 w + j of a chunk on lane j of warp w), then the xor tree of each warp, the 8 warps in index order, and
    k_align_step the C slots in index order"""
    v = np.asarray(v, dtype=np.float64)
    n = len(v)
    Cs = slots(n)
    rows = np.concatenate([v, np.zeros(-n % THREADS)]).reshape(-1, THREADS) if n else np.zeros((0, THREADS))
    idx = np.arange(32)
    total = 0.0
    for c in range(Cs):
        acc = np.zeros(THREADS)
        for r in range(c, len(rows), Cs):
            acc = acc + rows[r]
        s = 0.0
        for w in range(THREADS // 32):
            lanes = acc[32 * w:32 * w + 32]
            for o in (16, 8, 4, 2, 1):
                lanes = lanes + lanes[idx ^ o]
            s += float(lanes[0])
        total += s
    return total


def sums(ko, om, src, T, tau):
    """the 11 sums of k_align_eval at pose T: {inliers, sum |r|^2, JTJ 00, 01, 02, 11, 12, 22, JTr 0, 1, 2}, and the per-point
    distances"""
    src = np.ascontiguousarray(src, dtype=np.float64).reshape(-1, 3)
    n = len(src)
    if n == 0:
        return [0.0] * 11, np.zeros(0)
    T = np.asarray(T, dtype=np.float64)
    q = ko.se3_transform(T, src)
    nb, d = om.nearest(q)
    inl = d < tau
    with np.errstate(invalid="ignore", over="ignore"):  # non-finite points: their terms are masked out
        qx, qy, qz, qw = (float(v) for v in T[:4])
        r = q - nb
        rx, ry, rz = r[:, 0], r[:, 1], r[:, 2]
        ax, ay, az = _quat_rotate(qx, qy, qz, qw, 1.0, 0.0, 0.0)
        bx, by, bz = _quat_rotate(qx, qy, qz, qw, 0.0, 1.0, 0.0)
        cx, cy, cz = _quat_rotate(qx, qy, qz, qw, -src[:, 1], src[:, 0], np.zeros(n))
        one = np.ones(n)
        terms = [one, rx * rx + ry * ry + rz * rz, (ax * ax + ay * ay + az * az) * one, (ax * bx + ay * by + az * bz) * one,
                 ax * cx + ay * cy + az * cz, (bx * bx + by * by + bz * bz) * one, bx * cx + by * cy + bz * cz, cx * cx + cy * cy + cz * cz,
                 ax * rx + ay * ry + az * rz, bx * rx + by * ry + bz * rz, cx * rx + cy * ry + cz * rz]
        return [kernel_sum(np.where(inl, t, 0.0)) for t in terms], d


def align(ko, om, src, T0, tau, max_iterations=10, convergence=1e-3):
    """One alignment from T0: dict(traj=[pose after each of the max_iterations steps (unchanged once stopped)], statuses=[status after
    each], pose, status, iterations, last_step, v=the 11 sums at pose, n)"""
    T = [float(v) for v in T0]
    status, it, last, done = MAX_ITERATIONS, 0, 0.0, False
    traj, statuses = [], []
    for _ in range(max_iterations):
        if not done:
            v, _ = sums(ko, om, src, T, tau)
            N = v[0]
            if not N > 0.0:
                status, done = NO_CORRESPONDENCES, True
            else:
                dx = solve([x / N for x in v[2:8]], [x / N for x in v[8:11]])
                if dx is None:
                    status, done = SINGULAR, True
                else:
                    T = update(T, dx)
                    it += 1
                    last = step_norm(dx)
                    if last < convergence:
                        status, done = CONVERGED, True
        traj.append(list(T))
        statuses.append(status)
    v, _ = sums(ko, om, src, T, tau)
    return dict(traj=traj, statuses=statuses, pose=T, status=status, iterations=it, last_step=last, v=v,
                n=len(np.asarray(src).reshape(-1, 3)))


def check_alignment(a, res, where=""):
    """a returned kicp_planar_alignment (Alignment, or PlanarAlignment-like with the same field names) == the oracle's, bit for bit"""
    assert np.array_equal(np.asarray(a.pose[:], dtype=np.float64), np.asarray(res["pose"])), (where, list(a.pose), res["pose"])
    assert (a.status, a.iterations) == (res["status"], res["iterations"]), (where, a.status, a.iterations, res["status"], res["iterations"])
    assert a.last_step == res["last_step"], (where, a.last_step, res["last_step"])
    v, n = res["v"], res["n"]
    assert a.n_inliers == int(v[0]) and a.sum_sq == v[1], (where, a.n_inliers, a.sum_sq, v[:2])
    assert list(a.jtj) == v[2:8] and list(a.jtr) == v[8:11], (where, list(a.jtj), list(a.jtr), v[2:])
    assert a.fitness == (v[0] / n if n else 0.0)
    assert a.inlier_rmse == (math.sqrt(v[1] / v[0]) if v[0] > 0 else 0.0)
