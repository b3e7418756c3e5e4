"""The pose search, timed on one GPU.

cfg4's 1 001 499-point map (voxel 0.5 m) and its scan taken every k-th point (about 2k and about 8k points), searched with a 0.15 m gate from a prior
perturbed from the scan's true pose by a known planar offset, on two grids:
- start-up: +-4 m, +-pi, 0.5 m / 0.1 rad steps, 4 levels, keep 8;
- near-prior: +-1 m, +-0.2 rad, 0.1 m / 0.02 rad steps, 3 levels, keep 8.
Each case is timed as whole synchronous calls (host clock; every call ends in its synchronisation), in rounds that alternate the
cases, and reports the fastest and median ms per call, the hypotheses scored, point-hypothesis queries per second (points x
hypotheses / median time) and the recovered error against the offset that undoes the perturbation.  The workaround a caller has today,
Correspondences on device points once per level-0 hypothesis of the near-prior grid, is timed once per size for comparison.

Prints the card's name and power limit (read in the same run) and one JSON line.

    python scripts/pose_search_bench.py [--rounds 5]
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

TAU = 0.15  # the inlier gate of the search: a few finest steps wide (DESIGN.md §5)
GRIDS = {"startup": ((4.0, 4.0, math.pi), (0.5, 0.5, 0.1), 4), "near": ((1.0, 1.0, 0.2), (0.1, 0.1, 0.02), 3)}
PERTURB = {"startup": (1.37, -2.21, 0.83), "near": (0.37, -0.23, 0.041)}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def planar_inverse(x, y, yaw):
    c, s = math.cos(-yaw), math.sin(-yaw)
    return np.array([-(c * x - s * y), -(s * x + c * y), -yaw])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch

    import kinematic_icp_b200 as kb
    from oracle import kicp_oracle_py as ko
    from oracle import workloads as W

    w = W.Workload(4)
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, w.voxel_size, w.max_range, w.max_points_per_voxel)
    gm.load_voxels(*w.map.export_voxels())
    srcs = {n: np.ascontiguousarray(w.scan[:: len(w.scan) // n]) for n in (2000, 8000)}
    cases = [(g, n) for g in GRIDS for n in srcs]
    priors = {g: ko.se3_compose(w.true_pose, ko.planar_pose(*PERTURB[g])) for g in GRIDS}
    times = {c: [] for c in cases}
    out = {}
    for c in cases:  # warm-up: every shape once
        g, n = c
        he, st, lv = GRIDS[g]
        gm.PoseSearch(srcs[n], priors[g], TAU, he, st, levels=lv, keep=8)
    for r in range(args.rounds):
        for c in (cases if r % 2 == 0 else cases[::-1]):
            g, n = c
            he, st, lv = GRIDS[g]
            t0 = time.perf_counter()
            hyps, scored = gm.PoseSearch(srcs[n], priors[g], TAU, he, st, levels=lv, keep=8)
            times[c].append((time.perf_counter() - t0) * 1e3)
            fine = np.array(st) / 2 ** (lv - 1)
            err = np.abs(np.array(hyps[0].offset) - planar_inverse(*PERTURB[g]))
            out[c] = dict(scored=scored, err=[float(e) for e in err], within_one_fine_step=bool((err <= fine).all()),
                          inliers=hyps[0].n_inliers, n=len(srcs[n]))
    res = {}
    for c in cases:
        t = sorted(times[c])
        med = t[len(t) // 2]
        o = out[c]
        res["%s_%d" % c] = dict(ms_min=round(t[0], 3), ms_median=round(med, 3), hypotheses=o["scored"],
                                queries_per_s=o["n"] * o["scored"] / (med * 1e-3), err_xy_yaw=o["err"],
                                within_one_fine_step=o["within_one_fine_step"], best_inliers=o["inliers"], points=o["n"])
    # the workaround: one Correspondences call per level-0 hypothesis of the near-prior grid, device points, device outputs
    he, st, lv = GRIDS["near"]
    k = [int(math.floor(he[a] / st[a])) for a in range(3)]
    for n, src in srcs.items():
        dev = torch.from_numpy(src).cuda()
        outs = (torch.empty((len(src), 3), dtype=torch.float64, device="cuda"), torch.empty(len(src), dtype=torch.float64, device="cuda"),
                torch.empty(len(src), dtype=torch.uint8, device="cuda"))
        poses = [ko.se3_compose(priors["near"], ko.planar_pose(ix * st[0], iy * st[1], ip * st[2]))
                 for ip in range(-k[2], k[2] + 1) for ix in range(-k[0], k[0] + 1) for iy in range(-k[1], k[1] + 1)]
        gm.Correspondences(dev, poses[0], TAU, out=outs)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for p in poses:
            gm.Correspondences(dev, p, TAU, out=outs)
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) * 1e3
        res["workaround_near_%d" % n] = dict(ms=round(dt, 3), hypotheses=len(poses), ms_per_hypothesis=round(dt / len(poses), 4))
    gm.close()
    ctx.close()
    print("card: %s" % card())
    print(json.dumps(dict(bench="pose_search", card=card(), map_points=int(w.map.num_points()), results=res)))


if __name__ == "__main__":
    main()
