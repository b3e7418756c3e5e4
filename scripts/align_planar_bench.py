"""The planar alignment, timed on one GPU.

cfg4's 1 001 499-point map (voxel 0.5 m) and its scan taken every k-th point (about 2k and about 8k points), with the pose search's
near-prior setup of DESIGN.md §5: a prior perturbed from the true pose by (0.37, -0.23, 0.041 rad), PoseSearch on +-1 m, +-0.2 rad,
0.1 m / 0.02 rad steps, 3 levels, keep 8, gate 0.15 m.  AlignPlanar (gate 0.15 m, the reference's 10 iterations and 1e-3 convergence)
then starts from the best hypothesis (1 start) or from all 8 kept ones (8 starts).

- Each (points, starts) case is timed as whole synchronous calls (host clock; every call ends in its synchronisation), in rounds that
  alternate the cases, and reports the fastest and median ms per call and the iteration counts.
- The error per axis (|x|, |y|, |yaw| of truth^-1 * pose) after PoseSearch alone and after PoseSearch + AlignPlanar of the 8 kept
  hypotheses, the result picked by (stopped normally, more inliers, smaller sum_sq).
- The workaround a caller has without AlignPlanar: a host loop of Correspondences(points, pose) with the matched points returned, a
  3 x 3 numpy solve and the pose update, per iteration per start, timed for the same cases.

Prints the card's name and power limit (read in the same run) and one JSON line.

    python scripts/align_planar_bench.py [--rounds 7]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "kinematic-icp_b200", "python")):
    sys.path.insert(0, p)

TAU = 0.15
GRID = ((1.0, 1.0, 0.2), (0.1, 0.1, 0.02), 3)
PERTURB = (0.37, -0.23, 0.041)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def planar_error(ko, pose, truth):
    d = ko.se3_compose(ko.se3_inverse(truth), np.asarray(pose, dtype=np.float64))
    return [abs(float(d[4])), abs(float(d[5])), abs(2.0 * math.atan2(d[2], d[3]))]


def update(T, dx):
    """T * Delta(dx) as AlignPlanar applies it (q = normalize((0, 0, dx2 / 2, 1)))"""
    ax, ay, az, aw = T[:4]
    bz = dx[2] / 2.0
    q = np.array([ax + ay * bz, ay - ax * bz, az + aw * bz, aw - az * bz])
    q /= np.linalg.norm(q)
    v = np.array([dx[0], dx[1], 0.0])
    u = 2.0 * np.cross(T[:3], v)
    t = np.asarray(T[4:]) + v + aw * u + np.cross(T[:3], u)
    return np.r_[q, t]


def workaround(gm, src, T0, tau, iters=10, conv=1e-3):
    """the host loop: Correspondences at T, J^T J / J^T r in numpy, a 3 x 3 solve, the update; returns (pose, iterations)"""
    T = np.asarray(T0, dtype=np.float64)
    it = 0
    for _ in range(iters):
        nb, dist, inl, st = gm.Correspondences(src, T, tau)
        m = inl.astype(bool)
        if not m.any():
            break
        p = src[m]
        x, y, z, w = T[:4]
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                      [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        q = p @ R.T + T[4:]
        r = q - nb[m]
        c = np.stack([-p[:, 1], p[:, 0], np.zeros(len(p))], 1) @ R.T
        J = np.stack([np.broadcast_to(R[:, 0], c.shape), np.broadcast_to(R[:, 1], c.shape), c], 2)  # (k, 3, 3)
        A = np.einsum("kia,kib->ab", J, J) / len(p)
        b = np.einsum("kia,ki->a", J, r) / len(p)
        dx = -np.linalg.solve(A, b)
        T = update(T, dx)
        it += 1
        if np.linalg.norm(dx) < conv:
            break
    return T, it


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    import kinematic_icp_b200 as kb
    from oracle import kicp_oracle_py as ko
    from oracle import workloads as W

    w = W.Workload(4)
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, w.voxel_size, w.max_range, w.max_points_per_voxel)
    gm.load_voxels(*w.map.export_voxels())
    srcs = {n: np.ascontiguousarray(w.scan[:: len(w.scan) // n]) for n in (2000, 8000)}
    prior = ko.se3_compose(w.true_pose, ko.planar_pose(*PERTURB))
    he, st, lv = GRID
    ok = (kb._capi.KICP_ALIGN_CONVERGED, kb._capi.KICP_ALIGN_MAX_ITERATIONS)
    res, starts = {}, {}
    for n, src in srcs.items():
        hyps, _ = gm.PoseSearch(src, prior, TAU, he, st, levels=lv, keep=8)
        starts[n] = {1: np.array([hyps[0].pose]), 8: np.array([h.pose for h in hyps])}
        al = gm.AlignPlanar(src, starts[n][8], TAU)
        best = min(al, key=lambda a: (a.status not in ok, -a.n_inliers, a.sum_sq))
        res["error_%d" % n] = dict(search=planar_error(ko, hyps[0].pose, w.true_pose), search_align=planar_error(ko, best.pose, w.true_pose),
                                   finest_step=[s / 2 ** (lv - 1) for s in st], statuses=[a.status for a in al],
                                   iterations=[a.iterations for a in al], best_inliers=best.n_inliers, points=len(src))
    cases = [(n, k) for n in srcs for k in (1, 8)]
    for c in cases:  # warm-up: every shape once
        gm.AlignPlanar(srcs[c[0]], starts[c[0]][c[1]], TAU)
    times = {c: [] for c in cases}
    iters = {}
    for r in range(args.rounds):
        for c in (cases if r % 2 == 0 else cases[::-1]):
            n, k = c
            t0 = time.perf_counter()
            al = gm.AlignPlanar(srcs[n], starts[n][k], TAU)
            times[c].append((time.perf_counter() - t0) * 1e3)
            iters[c] = [a.iterations for a in al]
    for c in cases:
        t = sorted(times[c])
        res["align_%d_x%d" % c] = dict(ms_min=round(t[0], 3), ms_median=round(t[len(t) // 2], 3), iterations=iters[c],
                                       points=len(srcs[c[0]]), starts=c[1])
    for c in cases:  # the workaround, once per case after one warm-up call
        n, k = c
        workaround(gm, srcs[n], starts[n][k][0], TAU, iters=1)
        t0 = time.perf_counter()
        out = [workaround(gm, srcs[n], T0, TAU) for T0 in starts[n][k]]
        dt = (time.perf_counter() - t0) * 1e3
        total_it = sum(i for _, i in out)
        res["workaround_%d_x%d" % c] = dict(ms=round(dt, 3), iterations=[i for _, i in out],
                                            ms_per_iteration=round(dt / max(total_it, 1), 4))
    gm.close()
    ctx.close()
    print("card: %s" % card())
    print(json.dumps(dict(bench="align_planar", card=card(), map_points=int(w.map.num_points()), results=res)))


if __name__ == "__main__":
    main()
